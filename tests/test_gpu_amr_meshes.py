"""GPU tests of the multi-level device path (csrc/amr_ops.cu, csrc/amr_fast.cu, the host plan of csrc/amr_plan.cpp, the
enqueued step) on generated meshes (tests/amr_meshes.py): level jumps at every wall and corner, rectangular domains, meshes
of 1-5 blocks, every block order, both kernel modes.  Against the oracle (oracle/cup2d_amr_oracle.py, tests/amr_adapt_oracle.py),
which is pinned bit for bit on the reference's own mesh; the step is composed from the oracle with the oracle's own Poisson
assembly.

The one-level meshes of 1023 .. 4097 blocks and the multi-level mesh above 8192 blocks run the one-CTA reductions of the
enqueued step (amr_dt_kernel: 1024 threads striding over the per-block maxima; amr_wmean_kernel: four strided blocks per
thread, 4096 blocks a pass) across their pass boundaries.  A strided loop that skipped a block or stopped a pass early would
fail both checks there: the dt of a velocity whose maximum sits in the first block, the last block, block 1024 m or the last
block of a 4096-block pass would no longer be the host rule's; and the two pressure means would miss the blocks of the last
pass, so that the pressure change of a step would no longer have a zero h^2-weighted mean (off by about 1/nb relative).

They also pass on the CPU against the emulated build of the same sources (tools/run_emulated_gpu_tests.sh; a subset in
tests/test_amr_meshes_emulation.py)."""
import functools
import math

import numpy as np
import pytest
import scipy.sparse as sp

import amr_adapt_oracle as ado
import amr_meshes as M
import cup2d_amr_oracle as ao

pytestmark = [pytest.mark.gpu]

CASES = {**M.GENERATED, **M.TINY}
MESH_ORDERS = [(n, o) for n in CASES for o in M.ORDERS]
H0, NU, DT = 1 / 8, 1e-3, 1e-3
FAST = [pytest.param(False, id="base"), pytest.param(True, id="fast")]


WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    """the largest relative error seen per check, printed at the end of the module (visible with -s)"""
    yield
    for k, v in sorted(WORST.items()):
        print("WORST %-28s %.3e" % (k, v))


def rel(a, b, check=None):
    e = np.abs(a - b).max() / np.abs(b).max()
    if check:
        WORST[check] = max(WORST.get(check, 0.0), float(e))
    return e


def _perm(name, order):
    """the ordered list as indices into the sorted list"""
    bx, by, blocks, _ = CASES[name]
    s = {tuple(x): q for q, x in enumerate(M.order(blocks, bx, by, "sorted").tolist())}
    return np.array([s[tuple(x)] for x in M.order(blocks, bx, by, order).tolist()])


@functools.lru_cache(maxsize=None)
def _case(name):
    """seeded fields on the sorted list and the oracle's operators and RK2 stage on them"""
    bx, by, blocks, lmax = CASES[name]
    b = M.order(blocks, bx, by, "sorted")
    mesh = ao.Mesh(b, bx, by)
    nb = len(b)
    rng = np.random.default_rng(100 + nb)
    f = {"vel": rng.uniform(-1, 1, (nb, 8, 8, 2)), "pres": rng.uniform(-1, 1, (nb, 8, 8, 1)),
         "chi": rng.uniform(0, 1, (nb, 8, 8, 1)), "udef": rng.uniform(-1, 1, (nb, 8, 8, 2))}
    out = ao.amr_operators(mesh, H0, f["vel"], f["pres"], f["chi"], f["udef"], NU, DT)
    out["rhs0"] = ao.amr_pressure_rhs(mesh, H0, f["vel"], f["udef"], f["chi"], DT)
    dt = ao.amr_compute_dt(mesh, H0, f["vel"], NU, 0.5)
    out["step_dt"], out["rk2"] = dt, ao.amr_rk2(mesh, H0, f["vel"], NU, dt)
    return f, out


def _sim(blocks, bx, by, fast=False):
    from cup2d_b200.amr import AmrSimulation
    s = AmrSimulation(blocks, bx, by, H0, NU)
    s.set_fast(fast)
    return s


def _device_operators(name, order, fast):
    bx, by, blocks, _ = CASES[name]
    f, _ = _case(name)
    p = _perm(name, order)
    sim = _sim(M.order(blocks, bx, by, order), bx, by, fast)
    got = {}
    sim.upload("vel", f["vel"][p])
    sim.advect_diffuse_rhs(DT)
    got["adv"] = sim.download("tmpV")
    for lap, key in ((False, "rhs0"), (True, "rhs1")):
        sim.upload("tmpV", f["udef"][p])
        sim.upload("chi", f["chi"][p])
        sim.upload("pold", f["pres"][p])
        sim.pressure_rhs(DT, with_laplacian=lap)
        got[key] = sim.download("tmp")
    sim.upload("pres", f["pres"][p])
    sim.pressure_gradient(DT)
    got["gradp"] = sim.download("tmpV")
    sim.close()
    return got


@pytest.mark.parametrize("fast", FAST)
@pytest.mark.parametrize("name,order", MESH_ORDERS)
def test_operators_match_the_oracle(name, order, fast):
    """advect-diffuse (tmpV), pressure rhs without and with the Laplacian of pold (tmp), pressure gradient (tmpV)"""
    _, want = _case(name)
    p = _perm(name, order)
    got = _device_operators(name, order, fast)
    for key in ("adv", "rhs0", "rhs1", "gradp"):
        assert rel(got[key], want[key][p], "operators " + key) <= 1e-12, key


@pytest.mark.parametrize("fast", FAST)
@pytest.mark.parametrize("name", list(CASES))
def test_operators_do_not_depend_on_the_block_order(name, fast):
    """the operators of a shuffled list are those of the sorted list, permuted: bitwise on every block whose neighbours are
    all at its own level.  Next to a level jump the order of a ghost cell's sum follows the block numbering by design: a row
    of the plan's ghost tables (csrc/amr_plan.cpp, LC) lists its source cells sorted by (source block, cell), and the lab
    fill of the baseline and the fast kernels adds them in that order, so those blocks (AmrPlan.irregular) agree to rounding."""
    from cup2d_b200.amr import AmrPlan
    bx, by, blocks, _ = CASES[name]
    s = M.order(blocks, bx, by, "sorted")
    plan = AmrPlan(s, bx, by)
    irregular = np.zeros(len(s), dtype=bool)
    irregular[plan.irregular()] = True
    plan.close()
    base = _device_operators(name, "sorted", fast)
    for order in M.ORDERS[1:]:
        p = _perm(name, order)
        got = _device_operators(name, order, fast)
        for key, a in got.items():
            w = base[key][p]
            reg = ~irregular[p]
            assert np.array_equal(a[reg], w[reg]), (order, key)
            assert rel(a, w, "order invariance") <= 1e-14, (order, key)


def _tag_fields(name):
    """the seeded velocity and a chi that is nonzero in every fifth block only, so that the chi rule fires on some blocks"""
    f, _ = _case(name)
    nb = len(f["vel"])
    chi = np.zeros((nb, 8, 8, 1))
    chi[::5] = f["chi"][::5]
    chi[::5][chi[::5] < 0.7] = 0.0
    return f["vel"], chi


def _thresholds(linf):
    """(rtol, ctol) from the vorticity maxima of the blocks (the chi rule puts 2 rtol into the blocks it fires on): in the
    widest gaps between maxima in the upper and the lower half, each at least 1e-6 relative away from every maximum"""
    v = np.unique(linf)
    if len(v) < 4:
        return 0.5 * (v.max() + v.min()) if len(v) > 1 else 2 * v.max() + 1.0, 0.5 * v.min()
    half = len(v) // 2
    gaps = np.diff(v)
    hi = half + np.argmax(gaps[half:])
    lo = np.argmax(gaps[:half])
    rtol, ctol = 0.5 * (v[hi] + v[hi + 1]), 0.5 * (v[lo] + v[lo + 1])
    for t in (rtol, ctol):
        assert np.abs(v - t).min() >= 1e-6 * t
    return rtol, ctol


@pytest.mark.parametrize("name,order", MESH_ORDERS)
def test_adapt_tags_match_the_oracle(name, order):
    bx, by, blocks, lmax = CASES[name]
    vel, chi = _tag_fields(name)
    s = M.order(blocks, bx, by, "sorted")
    rtol, ctol = _thresholds(ao.amr_adapt_tags(ao.Mesh(s, bx, by), H0, vel, 0 * chi, 1.0, lmax)[1])
    want, wl = ao.amr_adapt_tags(ao.Mesh(s, bx, by), H0, vel, chi, rtol, lmax)
    p = _perm(name, order)
    sim = _sim(M.order(blocks, bx, by, order), bx, by)
    sim.upload("vel", vel[p])
    sim.upload("chi", chi[p])
    linf = sim.adapt_tags(rtol, lmax)
    field = sim.download("tmp").reshape(-1, 8, 8)
    sim.close()
    assert rel(field, want[p], "tagging field") <= 1e-12
    assert np.abs(linf - wl[p]).max() <= 1e-12 * wl.max()
    assert np.array_equal(linf > rtol, wl[p] > rtol) and np.array_equal(linf < ctol, wl[p] < ctol)
    if len(s) > 8:
        assert 0 < (wl > rtol).sum() < len(s) and (wl < ctol).any()


@pytest.mark.parametrize("name,order", MESH_ORDERS)
def test_dump_equals_the_oracle_byte_for_byte(name, order, tmp_path):
    bx, by, blocks, _ = CASES[name]
    f, _ = _case(name)
    b = M.order(blocks, bx, by, order)
    vel = f["vel"][_perm(name, order)]
    sim = _sim(b, bx, by)
    sim.upload("vel", vel)
    pref = str(tmp_path / "vel")
    sim.dump(0.25, pref)
    sim.close()
    xyz, attr = ao.amr_dump_arrays(ao.Mesh(b, bx, by), H0, vel)
    assert np.fromfile(pref + ".xyz.raw", dtype=np.float32).tobytes() == xyz.tobytes()
    assert np.fromfile(pref + ".attr.raw", dtype=np.float32).tobytes() == attr.tobytes()


REGRID_FIELDS = (("vel", "vector"), ("vold", "vector"), ("pres", "scalar"), ("pold", "scalar"), ("chi", "scalar"))


@pytest.mark.parametrize("order", ["reference", "random"])
@pytest.mark.parametrize("name", list(M.GENERATED))
def test_adapt_decision_and_transfer_match_the_oracle(name, order):
    """adapt() on the device: the decision and the new list follow the reference (fill_pos / Encode).  Both sides decide from
    the tags alone and sort the new list by Encode, so a shuffled list must give the same new mesh as the reference's order.
    The transferred fields against the oracle's transfer as in tests/test_gpu_amr_regrid.py (tmp holds the tagging field
    the device computed itself and is not compared)."""
    bx, by, blocks, lmax = CASES[name]
    vel, chi = _tag_fields(name)
    b = M.reference_order(blocks, bx, by, lmax) if order == "reference" else M.order(blocks, bx, by, order)
    s = M.order(blocks, bx, by, "sorted")
    p = np.array([{tuple(x): q for q, x in enumerate(s.tolist())}[tuple(x)] for x in b.tolist()])
    mesh = ao.Mesh(b, bx, by)
    rtol, ctol = _thresholds(ao.amr_adapt_tags(mesh, H0, vel[p], 0 * chi[p], 1.0, lmax)[1])
    _, wl = ao.amr_adapt_tags(mesh, H0, vel[p], chi[p], rtol, lmax)
    want_blocks = ado.amr_adapt_mesh(mesh, wl, rtol, ctol, lmax)
    rng = np.random.default_rng(len(b))
    f = {"vel": vel[p], "vold": rng.uniform(-1, 1, vel.shape), "pres": rng.uniform(-1, 1, chi.shape),
         "pold": rng.uniform(-1, 1, chi.shape), "chi": chi[p]}
    sim = _sim(b, bx, by)
    for n, a in f.items():
        sim.upload(n, a)
    assert sim.adapt(rtol, ctol, lmax)
    assert np.array_equal(sim.blocks, want_blocks)
    new = np.asarray(want_blocks)
    assert any((l - 1, i // 2, j // 2) in mesh.index for l, i, j in new.tolist())          # something was refined
    want = ado.amr_regrid(mesh, new, {n: (f[n], k) for n, k in REGRID_FIELDS})
    got = {n: sim.download(n) for n, _ in REGRID_FIELDS}
    sim.close()
    _check_transfer(want, got, b, new, bx, by)


def _check_transfer(want, got, blocks, new_blocks, bx, by):
    """copied and compressed blocks bitwise; refined blocks bitwise where the parent's lab rows are plain copies, else to
    1e-13 (the rounding of the flattened ghost sums), as in tests/test_gpu_amr_regrid.py"""
    from test_gpu_amr_regrid import _exact_parents
    old = {tuple(x): k for k, x in enumerate(np.asarray(blocks).tolist())}
    exact = {"vector": _exact_parents(blocks, bx, by, 4), "scalar": _exact_parents(blocks, bx, by, 5)}
    for n, kind in REGRID_FIELDS:
        a, w = got[n], want[n]
        for q, (l, i, j) in enumerate(np.asarray(new_blocks).tolist()):
            parent = old.get((l - 1, i // 2, j // 2))
            if (l, i, j) in old or parent is None or exact[kind][parent]:
                assert np.array_equal(a[q], w[q]), (n, q)
            else:
                assert np.abs(a[q] - w[q]).max() <= 1e-13 * np.abs(w).max(), (n, q)


def _oracle_step(name, order, max_iter):
    """the step composed from the oracle: its dt rule, RK2, rhs (x0 = 0), BiCGSTAB on its own Poisson assembly in this block
    order, the pressure correction"""
    import cup2d_oracle as orc
    bx, by, blocks, _ = CASES[name]
    f, out = _case(name)
    p = _perm(name, order)
    b = M.order(blocks, bx, by, order)
    mesh = ao.Mesh(b, bx, by)
    nb = len(b)
    dt = out["step_dt"]
    assert dt == ao.amr_compute_dt(mesh, H0, f["vel"][p], NU, 0.5)
    v = out["rk2"][p]
    rhs, pold, p0 = ao.amr_poisson_rhs(mesh, H0, v, np.zeros_like(v), np.zeros((nb, 8, 8, 1)), f["pres"][p], dt)
    r, c, val = ao.amr_poisson_matrix(mesh)
    A = sp.coo_matrix((val, (r, c)), shape=(64 * nb, 64 * nb)).tocsr()
    P = orc.build_P_inv()
    x, it, _ = orc.bicgstab(rhs.reshape(-1), p0.reshape(-1), max_iter=max_iter, A=lambda q: A @ q,
                            M=lambda q: (q.reshape(nb, 64) @ P.T).reshape(-1))
    vel, pres = ao.amr_pressure_correct(mesh, H0, v, x.reshape(nb, 8, 8, 1), pold, dt)
    return dt, it, vel, pres


def _step_sim(name, order, fast):
    bx, by, blocks, _ = CASES[name]
    f, _ = _case(name)
    p = _perm(name, order)
    sim = _sim(M.order(blocks, bx, by, order), bx, by, fast)
    sim.upload("vel", f["vel"][p])
    sim.upload("pres", f["pres"][p])
    sim.upload("chi", np.zeros_like(f["pres"]))
    return sim


@pytest.mark.parametrize("fast", FAST)
@pytest.mark.parametrize("name,order", MESH_ORDERS)
def test_step_matches_the_composed_oracle(name, order, fast):
    sim = _step_sim(name, order, fast)
    dt, it, _ = sim.step(cfl=0.5, max_iter=12)
    vel, pres = sim.download("vel"), sim.download("pres")
    sim.close()
    want_dt, want_it, want_vel, want_pres = _oracle_step(name, order, 12)
    assert dt == want_dt
    assert it == want_it == 12
    assert rel(vel, want_vel, "step vel") <= 1e-9 and rel(pres, want_pres, "step pres") <= 1e-9


@pytest.mark.parametrize("fast", FAST)
@pytest.mark.parametrize("name,order", MESH_ORDERS)
def test_enqueued_step_matches_the_blocking_step(name, order, fast):
    a, b = _step_sim(name, order, fast), _step_sim(name, order, fast)
    ra = a.step(cfl=0.5, max_iter=12)
    b.step_enqueue(cfl=0.5, max_iter=12)
    rb = b.step_result()
    assert rb[0] == ra[0] and rb[1] == ra[1]
    for n in ("vel", "pres"):
        assert rel(b.download(n), a.download(n), "enqueued " + n) <= 1e-13, n
    a.close()
    b.close()


# ---- the reductions of the enqueued step across their pass boundaries ----------------------------------------------
BIG = {**M.COUNTS, **M.LARGE}


def _plant_sites(nb):
    """block indices (in list order) to hold the largest |u|: the first and the last block, block 1024 m and the last
    block of a 4096-block pass, where the mesh has them"""
    sites = {"first": 0, "last": nb - 1}
    if nb > 1024:
        sites["k1024"] = 1024 * ((nb - 1) // 1024)
    if nb > 4096:
        sites["pass4096"] = 4096 * ((nb - 1) // 4096) - 1
    return sites


DT_CASES = [(n, s) for n, c in BIG.items() for s in _plant_sites(len(c[2]))]


def _big_fields(name):
    bx, by, blocks, _ = BIG[name]
    b = M.order(blocks, bx, by, "random")
    rng = np.random.default_rng(len(b))
    return b, bx, by, rng.uniform(-0.5, 0.5, (len(b), 8, 8, 2)), rng.uniform(-1, 1, (len(b), 8, 8, 1))


@pytest.mark.parametrize("name,site", DT_CASES)
def test_device_dt_rule_sees_every_block(name, site):
    b, bx, by, vel, _ = _big_fields(name)
    k = _plant_sites(len(b))[site]
    vel[k, 3, 5, 1] = -2.75
    sim = _sim(b, bx, by, True)
    sim.upload("vel", vel)
    sim.upload("pres", np.zeros((len(b), 8, 8, 1)))
    sim.step_enqueue(cfl=0.5, max_iter=1)
    dt, _, _ = sim.step_result()
    sim.close()
    assert dt == ao.amr_compute_dt(ao.Mesh(b, bx, by), H0, vel, NU, 0.5)


@pytest.mark.parametrize("name", list(BIG))
def test_enqueued_pressure_means_cover_every_block(name):
    """x from 12 iterations on x0 = 0 is nonzero in every block; the enqueued correction makes the pressure change of the
    step, p - pold = x' - mean_h2(x'), free of h^2-weighted mean"""
    b, bx, by, vel, pres = _big_fields(name)
    sim = _sim(b, bx, by, True)
    sim.upload("vel", vel)
    sim.upload("pres", pres)
    sim.step_enqueue(cfl=0.5, max_iter=12)
    _, it, _ = sim.step_result()
    p = sim.download("pres")
    sim.close()
    assert it == 12
    h2 = (H0 / (1 << b[:, 0].astype(np.int64))) ** 2
    d = (p - pres).reshape(len(b), 64)
    assert (np.abs(d).max(axis=1) > 0).all()
    total = math.fsum((d * h2[:, None]).reshape(-1).tolist())
    scale = math.fsum((np.abs(d) * h2[:, None]).reshape(-1).tolist())
    WORST["pressure mean"] = max(WORST.get("pressure mean", 0.0), abs(total) / scale)
    assert abs(total) <= 1e-13 * scale, (total, scale)
