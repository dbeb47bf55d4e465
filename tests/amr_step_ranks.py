"""Enqueued time steps (cup2d_amr_step_enqueue / _pressure_enqueue / _step_result / _set_graph) on distributed multi-level
contexts (cup2d_amr_create_ranks): the cases and the per-rank runner shared by tests/test_amr_step_enqueue_ranks_emulation.py
(ranks as threads of one process, on the emulated library), tests/test_gpu_amr_step_enqueue_ranks.py (one H100, a one-rank
distributed context) and tools/multi_gpu_amr_enqueue_check.py (several GPUs, one process per GPU).

The meshes are those of tests/test_gpu_amr_step_graph.py: the reference's run.sh mesh (tests/golden/amrlab_lmax8.npz) and a
synthetic three-level mesh (tools/bench_amr.three_level_mesh(3, ...)) with seeded fields."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE, os.path.join(ROOT, "tools"), os.path.join(HERE, "golden")):
    if p not in sys.path:
        sys.path.insert(0, p)

from amr_bodies_ranks import ThreadDist, on_threads  # noqa: E402,F401  (re-exported for the tests)

MESHES = ("runsh", "synthetic")
FIELD_TOL = 1e-13


def mesh(name):
    """(blocks, bpdx, bpdy, h0, nu, vel, pres), as tests/test_gpu_amr_step_graph.py builds them"""
    if name == "runsh":
        d = np.load(os.path.join(HERE, "golden", "amrlab_lmax8.npz"))
        return d["blocks"], int(d["bpdx"]), int(d["bpdy"]), float(d["h0"]), float(d["nu"]), d["vel"], d["pres"]
    import bench_amr
    blocks = bench_amr.three_level_mesh(3, r1=0.3, r2=0.15, centre=(0.45, 0.55))
    h0 = 1 / 8
    rng = np.random.default_rng(11)
    vel, pres = bench_amr.seeded_fields(blocks, h0)
    return blocks, 1, 1, h0, 1e-3, vel + 0.05 * rng.uniform(-1, 1, vel.shape), pres + 0.05 * rng.uniform(-1, 1, pres.shape)


def level_cut(m, W):
    """rank_begin for W ranks, near-even, each cut moved onto a block with a coarse face neighbour before it, so that the
    fine and the coarse side of that level interface lie on different ranks"""
    from cup2d_b200.amr import AmrPlan
    blocks, bx, by = m[0], m[1], m[2]
    nb = len(blocks)
    plan = AmrPlan(blocks, bx, by)
    faces = plan.faces()           # (fine, face, coarse, face, half)
    plan.close()
    fine_after = np.unique(faces[faces[:, 2] < faces[:, 0], 0])
    rb = [0]
    for r in range(1, W):
        want = nb * r // W
        k = int(fine_after[np.argmin(np.abs(fine_after - want))])
        rb.append(k)
    rb.append(nb)
    rb = np.array(rb, dtype=np.int64)
    assert all(rb[r] < rb[r + 1] for r in range(W)), rb
    own = np.searchsorted(rb, np.arange(nb), side="right") - 1
    assert (own[faces[:, 0]] != own[faces[:, 2]]).any(), rb
    return rb


def make(m, rank=None, rb=None, dist=None, graph=True, device=0):
    """a plain fast-kernel context (rb None) or this rank's share of a distributed one, the mesh's fields uploaded"""
    from cup2d_b200.amr import AmrSimulation
    blocks, bx, by, h0, nu, vel, pres = m
    if rb is None:
        sim = AmrSimulation(blocks, bx, by, h0, nu, device=device)
        sim.set_fast(True)
        b0, b1 = 0, len(blocks)
    else:
        sim = AmrSimulation.distributed(blocks, bx, by, h0, nu, rank, rb, dist, device=device)
        b0, b1 = int(rb[rank]), int(rb[rank + 1])
    sim.set_graph(graph)
    sim.upload("vel", vel[b0:b1])
    sim.upload("pres", pres[b0:b1])
    return sim


def fields(sim):
    return {n: sim.download(n) for n in ("vel", "pres")}


def run_steps(sim, n, enqueued, check_dt=False, cfl=0.5, **kw):
    """n steps, enqueued (step_enqueue + step_result each) or blocking (step): [(dt, iterations, residual)], the fields
    after the last.  check_dt: before every enqueued step, the blocking dt rule (compute_dt) on the same velocity, which
    the step's dt must equal bit for bit"""
    out = []
    for _ in range(n):
        if enqueued:
            dt_host = sim.compute_dt(cfl)[1] if check_dt else None
            sim.step_enqueue(cfl=cfl, **kw)
            r = sim.step_result()
            assert dt_host is None or r[0] == dt_host, (r[0], dt_host)
        else:
            r = sim.step(cfl=cfl, **kw)
        out.append(r)
    return out, fields(sim)


def pressure_inputs(m, seed=5):
    """a shape on every third block: ids, chi [n,8,8], u_def [n,8,8,2], and the chi field [nb,8,8,1]"""
    nb = len(m[0])
    rng = np.random.default_rng(seed)
    ids = np.arange(0, nb, 3, dtype=np.int32)
    X, U = rng.uniform(0, 1, (len(ids), 8, 8)), rng.uniform(-0.5, 0.5, (len(ids), 8, 8, 2))
    chi = np.zeros((nb, 8, 8, 1))
    chi[ids] = X[..., None]
    return ids, X, U, chi


def pressure_section(sim, m, b0, b1, enqueued, dt=1e-3, **kw):
    """shape_set + udef_assemble on this rank's blocks, then the pressure section, enqueued or blocking: (iterations,
    residual, fields)"""
    ids, X, U, chi = pressure_inputs(m)
    mine = (ids >= b0) & (ids < b1)
    sim.upload("chi", chi[b0:b1])
    sim.shape_set(0, ids[mine] - b0, X[mine], U[mine])
    sim.udef_assemble()
    if enqueued:
        sim.pressure_enqueue(dt, **kw)
        _, it, err = sim.step_result()
    else:
        sim.poisson_rhs(dt)
        it, err = sim.poisson_solve(**kw)
        sim.pressure_correct(dt)
    return it, err, fields(sim)


def rel(got, want):
    return float(np.abs(got - want).max() / np.abs(want).max())


def joined(parts, name):
    """one field over all ranks, in block order"""
    return np.concatenate([p[name] for p in parts])
