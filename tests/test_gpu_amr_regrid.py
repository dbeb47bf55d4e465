"""GPU tests of the in-place regrid of multi-level contexts (cup2d_amr_regrid, csrc/amr_regrid.cu) and of the whole adapt()
chain (AmrSimulation.adapt): against the reference's own adapt() on its run.sh mesh (tests/golden/amrregrid_lmax8.npz), against
a freshly created context on the new mesh, and against the oracle on synthetic three-level meshes (compression included).
They also pass on the CPU against the emulated build of the same sources (tests/test_amr_regrid.py)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import amr_adapt_oracle as ao

pytestmark = [pytest.mark.gpu]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = (("vel", "vector"), ("vold", "vector"), ("pres", "scalar"), ("pold", "scalar"), ("chi", "scalar"), ("tmp", "scalar"))


@pytest.fixture(scope="module")
def g(golden_dir):
    sys.path.insert(0, golden_dir)
    import make_regrid_golden
    return make_regrid_golden.load(os.path.join(golden_dir, "amrregrid_lmax8.npz"))


def _sim(blocks, bpdx, bpdy, h0, fields):
    from cup2d_b200.amr import AmrSimulation
    sim = AmrSimulation(blocks, bpdx, bpdy, h0, 4e-5)
    for n, a in fields.items():
        sim.upload(n, a)
    return sim


def _exact_parents(blocks, bpdx, bpdy, which):
    """old blocks whose kind-`which` lab rows are all plain copies or wall reflections (one term of weight +-1): their
    children are bitwise the reference's; the others carry the rounding of the flattened ghost sums"""
    from cup2d_b200.amr import AmrPlan
    p = AmrPlan(blocks, bpdx, bpdy)
    rowptr, _, _, w = p.stencil(which)
    p.close()
    first = w[np.minimum(rowptr[:-1], len(w) - 1)]
    one = (np.diff(rowptr) == 1) & (np.abs(first) == 1.0)
    return one.reshape(len(blocks), -1).all(axis=1)


def _check_against(g_new, got, blocks, new_blocks, bpdx, bpdy):
    old = {tuple(b): k for k, b in enumerate(np.asarray(blocks).tolist())}
    exact = {4: _exact_parents(blocks, bpdx, bpdy, 4), 5: _exact_parents(blocks, bpdx, bpdy, 5)}
    nexact = 0
    for n, kind in FIELDS:
        a, w = got[n], g_new[n]
        scale = np.abs(w).max()
        for q, (l, i, j) in enumerate(np.asarray(new_blocks).tolist()):
            if (l, i, j) in old or (l - 1, i // 2, j // 2) not in old:   # copied or compressed: bitwise
                assert np.array_equal(a[q], w[q]), (n, q)
            elif exact[4 if kind == "vector" else 5][old[(l - 1, i // 2, j // 2)]]:
                assert np.array_equal(a[q], w[q]), (n, q)
                nexact += 1
            else:
                assert np.abs(a[q] - w[q]).max() <= 1e-13 * scale, (n, q)
    return nexact


def test_regrid_reproduces_the_reference_transfer(g):
    bx, by = int(g["bpdx"]), int(g["bpdy"])
    sim = _sim(g["blocks"], bx, by, float(g["h0"]), {n: g[n] for n, _ in FIELDS} | {"tmpV": np.random.default_rng(1).uniform(-1, 1, g["vel"].shape)})
    sim.regrid(g["new_blocks"])
    assert np.array_equal(sim.blocks, g["new_blocks"])
    got = {n: sim.download(n) for n, _ in FIELDS}
    _check_against({n: g["new_" + n] for n, _ in FIELDS}, got, g["blocks"], g["new_blocks"], bx, by)
    assert not sim.download("tmpV").any()
    sim.close()


@pytest.mark.parametrize("fast", [False, True])
def test_regridded_context_steps_like_a_fresh_one(g, fast):
    """a step of the regridded context is bitwise the step of a context created on the new mesh with the same fields"""
    bx, by, h0 = int(g["bpdx"]), int(g["bpdy"]), float(g["h0"])
    a = _sim(g["blocks"], bx, by, h0, {n: g[n] for n, _ in FIELDS})
    a.set_fast(fast)
    a.step(cfl=0.5, max_iter=3)    # tables, Poisson context and lab buffers of the old mesh exist before the regrid
    for n, _ in FIELDS:
        a.upload(n, g[n])
    a.regrid(g["new_blocks"])
    b = _sim(g["new_blocks"], bx, by, h0, {n: a.download(n) for n, _ in FIELDS} | {"tmpV": a.download("tmpV")})
    b.set_fast(fast)
    for _ in range(2):
        ra, rb = a.step(cfl=0.5, max_iter=5), b.step(cfl=0.5, max_iter=5)
        assert ra == rb
        for n in ("vel", "pres", "tmp"):
            assert np.array_equal(a.download(n), b.download(n)), n
    a.close()
    b.close()


def test_regrid_error_paths(g):
    from cup2d_b200 import lib as L
    bx, by = int(g["bpdx"]), int(g["bpdy"])
    sim = _sim(g["blocks"], bx, by, float(g["h0"]), {"vel": g["vel"]})
    lib, blocks = sim.lib, np.ascontiguousarray(g["blocks"])
    P = C.POINTER(C.c_int32)
    # unchanged mesh: a no-op
    assert lib.cup2d_amr_regrid(sim._h, len(blocks), blocks.ctypes.data_as(P)) == 0
    assert np.array_equal(sim.download("vel"), g["vel"])
    bad = []
    b2 = blocks.copy()                      # a block two levels finer
    b2[0] = [blocks[0, 0] + 2, 4 * blocks[0, 1], 4 * blocks[0, 2]]
    bad.append(b2)
    bad.append(blocks[1:].copy())           # a block missing
    new = np.ascontiguousarray(g["new_blocks"])
    bad.append(new[1:].copy())              # a refined parent with three children
    bad.append(np.concatenate([blocks, blocks[:1]]))   # a block twice
    for m in bad:
        m = np.ascontiguousarray(m, dtype=np.int32)
        assert lib.cup2d_amr_regrid(sim._h, len(m), m.ctypes.data_as(P)) == -1
        assert b"cup2d_amr_regrid" in lib.cup2d_last_error()
    assert np.array_equal(sim.download("vel"), g["vel"])     # untouched
    sim.regrid(g["new_blocks"])                               # still usable
    rb = np.array([0, len(g["new_blocks"]) // 2, len(g["new_blocks"])], dtype=np.int64)
    L.check(lib.cup2d_amr_set_ranks(sim._h, 0, 2, rb.ctypes.data_as(C.POINTER(C.c_int64))))
    assert lib.cup2d_amr_regrid(sim._h, len(blocks), blocks.ctypes.data_as(P)) == -4
    sim.close()


def test_adapt_chain_from_the_reference_state(g):
    """AmrSimulation.adapt(Rtol, Ctol, levelMax) on the pre-adapt state: the device's tags, the host decision, the device
    transfer give the reference's new mesh and fields (tmp, the tagging field the device computed itself, to rounding)"""
    bx, by = int(g["bpdx"]), int(g["bpdy"])
    sim = _sim(g["blocks"], bx, by, float(g["h0"]), {n: g[n] for n, _ in FIELDS if n != "tmp"})
    assert sim.adapt(float(g["rtol"]), float(g["ctol"]), int(g["level_max"]))
    assert np.array_equal(sim.blocks, g["new_blocks"])
    for n, _ in FIELDS:
        got, want = sim.download(n), g["new_" + n]
        tol = 1e-12 if n == "tmp" else 1e-13
        assert np.abs(got - want).max() <= tol * np.abs(want).max(), n
    sim.close()


@pytest.mark.parametrize("base", [3, 4])
def test_synthetic_three_level_regrid_vs_oracle(base):
    """refine and compress (three-level meshes have plateaus that can coarsen): the device against the oracle's transfer"""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import bench_amr
    from cup2d_b200.amr import adapt_mesh
    blocks = bench_amr.three_level_mesh(base, r1=0.3, r2=0.15, centre=(0.45, 0.55))
    h0, lmax = 1 / 8, base + 3
    rng = np.random.default_rng(base)
    vel, pres = bench_amr.seeded_fields(blocks, h0)
    f = {"vel": vel + 0.05 * rng.uniform(-1, 1, vel.shape), "vold": rng.uniform(-1, 1, vel.shape),
         "pres": pres + 0.05 * rng.uniform(-1, 1, pres.shape), "pold": rng.uniform(-1, 1, pres.shape),
         "chi": rng.uniform(0, 1, pres.shape), "tmp": rng.uniform(-1, 1, pres.shape)}
    groups = {}
    for l, i, j in blocks.tolist():   # one tag per sibling group, so that whole groups compress
        groups.setdefault((l, i // 2, j // 2), rng.uniform(0, 1))
    linf = np.array([groups[(l, i // 2, j // 2)] for l, i, j in blocks.tolist()])
    new = adapt_mesh(blocks, 1, 1, lmax, linf, 0.7, 0.35)
    mesh = ao.Mesh(blocks, 1, 1)
    kinds = dict(FIELDS)
    want = ao.amr_regrid(mesh, new, {n: (f[n], kinds[n]) for n in f})
    ncomp = sum((l + 1, 2 * i, 2 * j) in mesh.index for l, i, j in new.tolist())
    nref = sum((l - 1, i // 2, j // 2) in mesh.index for l, i, j in new.tolist())
    assert ncomp > 0 and nref > 0
    sim = _sim(blocks, 1, 1, h0, f)
    sim.regrid(new)
    assert _check_against(want, {n: sim.download(n) for n in f}, blocks, new, 1, 1) > 0
    sim.close()
