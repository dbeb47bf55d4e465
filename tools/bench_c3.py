"""BASELINE.json configs[2]-style measurement: 4096^2 uniform grid on one GPU, time steps whose Poisson solves stop on the
tolerance (poissonTol 1e-6; stopping rule cuda.cu:535-541, main.cpp:7028-7030) instead of after a fixed iteration count.

The whole step — dt control, RK2, right-hand side, the BiCGSTAB loop as a graph WHILE node whose condition the device sets,
best-iterate correction — is ONE graph launch; the host reads (dt, iterations, residual) once per step after the timed
region of that step.  Parity of this mode is tests/test_gpu_parity.py::test_tolerance_driven_steps_vs_oracle (256^2, vs the
numpy oracle) and ::test_graph_while_node_stops_where_the_host_polled_solve_stops.

  python tools/bench_c3.py [level=9] [steps=6] [tol=1e-6]      -> one JSON line
"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402  (CUDA events)

import cup2d_b200  # noqa: E402


def main():
    L = int(sys.argv[1]) if len(sys.argv) > 1 else 9
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 6
    tol = float(sys.argv[3]) if len(sys.argv) > 3 else 1e-6
    N = 8 << L
    sim = cup2d_b200.Simulation(L, nu=1e-4, cfl=0.5)
    order = sim.local_order
    bi = order[:, 0].astype(np.float64)[:, None, None]
    bj = order[:, 1].astype(np.float64)[:, None, None]
    ix = np.arange(8, dtype=np.float64)[None, None, :]
    iy = np.arange(8, dtype=np.float64)[None, :, None]
    X = (bi * 8 + ix + 0.5) / N
    Y = (bj * 8 + iy + 0.5) / N
    rng = np.random.default_rng(1234)
    u = np.sin(2 * np.pi * X) * np.cos(2 * np.pi * Y) + 0.01 * rng.uniform(-1, 1, X.shape)
    v = -np.cos(2 * np.pi * X) * np.sin(2 * np.pi * Y) + 0.01 * rng.uniform(-1, 1, X.shape)
    vel = np.ascontiguousarray(np.stack([u, v], axis=-1).reshape(-1))
    sim.upload_blocks("vel", vel)
    sim.upload_blocks("pres", np.zeros(order.shape[0] * 64))
    kw = dict(tol_abs=tol, tol_rel=0.0, max_restarts=0, max_iter=1000)
    stream = torch.cuda.ExternalStream(sim.stream, device=torch.device("cuda", 0))
    # warm-up: the first steps run kernel by kernel and capture the step graphs
    for _ in range(4):
        sim.step_enqueue(**kw)
        sim.step_result()
    rows = []
    with torch.cuda.stream(stream):
        for _ in range(steps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            sim.step_enqueue(**kw)
            e1.record(stream)
            dt, it, err = sim.step_result()
            e1.synchronize()
            rows.append({"ms": e0.elapsed_time(e1), "iters": int(it), "err": float(err), "dt": float(dt)})
    ms = float(np.mean([r["ms"] for r in rows]))
    iters = float(np.mean([r["iters"] for r in rows]))
    cells = N * N
    fixed = None
    # the same steps with the iteration count fixed to the mean: what the WHILE node and the device-side stop cost
    k = max(1, int(round(iters)))
    for _ in range(3):
        sim.step_enqueue(max_iter=k, max_restarts=0)
        sim.step_result()
    with torch.cuda.stream(stream):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(steps):
            sim.step_enqueue(max_iter=k, max_restarts=0)
        e1.record(stream)
        sim.step_result()
        e1.synchronize()
        fixed = e0.elapsed_time(e1) / steps
    print(json.dumps({
        "workload": f"{N}x{N} uniform grid (level {L}), Taylor-Green + perturbation, nu=1e-4, CFL=0.5, 1 GPU; Poisson solve stops at "
                    f"L-inf residual <= {tol:g} (BASELINE.json configs[2] setting)",
        "steps": steps, "ms_per_step": ms, "poisson_iters_per_step": iters, "residual_at_stop": max(r["err"] for r in rows),
        "ms_per_poisson_iteration_incl_rest_of_step": ms / max(iters, 1.0),
        "Mcell_updates_per_s": cells * (2 + iters) / (ms * 1e-3) / 1e6,
        "fixed_iteration_steps_ms": fixed, "fixed_iterations": k,
        "per_step": rows,
        "note": "one graph launch per step; the Krylov loop is a conditional WHILE node driven by the device-side `done` flag"}))
    sim.close()


if __name__ == "__main__":
    main()
