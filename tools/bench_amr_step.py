"""Needs a GPU (not part of bench.py's line): median wall time per multi-level step, blocking cup2d_amr_step against the
enqueued form (cup2d_amr_step_enqueue + cup2d_amr_step_result, replayed as a CUDA graph), fast kernels, on the reference's
run.sh mesh (tests/golden/amrlab_lmax8.npz) and on the synthetic three-level meshes of tools/bench_amr.py at base levels 5-9
(9 = config C5), each with 10 fixed Krylov iterations and with a tolerance-driven solve (tol_abs 1e-7, at most 100
iterations, so that C5 stays affordable).  The two forms alternate over
ROUNDS rounds in this one process, every timed step ends in a device synchronise, both are warmed up first.  Also: the host
time of one cup2d_amr_step_enqueue call, and at C5 the device time per step of both forms from CUDA events.
  python tools/bench_amr_step.py [max_base_level=9] [steps_per_round=10]
Prints one JSON line with the card's name and power limit."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np

ROUNDS = 3
SOLVES = {"fixed10": dict(max_iter=10), "tol1e-7_cap100": dict(tol_abs=1e-7, max_restarts=100, max_iter=100)}


def median_spread(xs):
    xs = np.asarray(xs)
    return {"median": float(np.median(xs)), "p10": float(np.percentile(xs, 10)), "p90": float(np.percentile(xs, 90))}


def bench_mesh(label, blocks, bx, by, h0, nu, vel, pres, steps, device_time):
    import torch
    from cup2d_b200.amr import AmrSimulation
    out = {"mesh": label, "blocks": int(len(blocks)), "levels": sorted(set(blocks[:, 0].tolist()))}
    for sname, kw in SOLVES.items():
        sims = {}
        for form in ("blocking", "enqueued"):
            s = AmrSimulation(blocks, bx, by, h0, nu)
            s.set_fast(True)
            s.upload("vel", vel)
            s.upload("pres", pres)
            sims[form] = s

        def one(form):
            s = sims[form]
            if form == "blocking":
                r = s.step(cfl=0.5, **kw)
            else:
                s.step_enqueue(cfl=0.5, **kw)
                r = s.step_result()
            torch.cuda.synchronize()
            return r

        for form in sims:            # warm-up: tables, Poisson context, the direct first enqueue and the graph capture
            for _ in range(3):
                one(form)
        wall = {f: [] for f in sims}
        iters = {f: [] for f in sims}
        for _ in range(ROUNDS):
            for form in sims:
                for _ in range(steps):
                    t0 = time.perf_counter()
                    r = one(form)
                    wall[form].append((time.perf_counter() - t0) * 1e3)
                    iters[form].append(r[1])
        res = {f: median_spread(wall[f]) | {"iters_median": float(np.median(iters[f]))} for f in sims}
        res["speedup_median"] = res["blocking"]["median"] / res["enqueued"]["median"]
        # host time of the enqueue call alone (graph launch), the device drained between calls
        e = sims["enqueued"]
        host = []
        for _ in range(steps):
            t0 = time.perf_counter()
            e.step_enqueue(cfl=0.5, **kw)
            host.append((time.perf_counter() - t0) * 1e3)
            e.step_result()
        res["enqueue_host_ms"] = median_spread(host)
        if device_time:              # device time per step from CUDA events on the context's stream (the same work)
            dev = {}
            for form in sims:
                ms = []
                for _ in range(steps):
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    torch.cuda.synchronize()
                    a.record()
                    one(form)
                    b.record()
                    b.synchronize()
                    ms.append(a.elapsed_time(b))
                dev[form] = median_spread(ms)
            res["event_ms"] = dev
        out[sname] = res
        for s in sims.values():
            s.close()
    return out


def main():
    import torch
    import bench_amr
    maxb = int(sys.argv[1]) if len(sys.argv) > 1 else 9
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 10
    props = torch.cuda.get_device_properties(0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    d = np.load(os.path.join(ROOT, "tests", "golden", "amrlab_lmax8.npz"))
    rows = [bench_mesh("run.sh lmax8", d["blocks"], int(d["bpdx"]), int(d["bpdy"]), float(d["h0"]), float(d["nu"]), d["vel"],
                       d["pres"], steps, False)]
    for base in range(5, maxb + 1):
        blocks = bench_amr.three_level_mesh(base)
        h0 = 1.0 / 8
        vel, pres = bench_amr.seeded_fields(blocks, h0)
        rows.append(bench_mesh(f"synthetic base {base}" + (" (C5)" if base == 9 else ""), blocks, 1, 1, h0, 1e-4, vel, pres,
                               steps, base == maxb))
    print(json.dumps({"tool": "bench_amr_step", "gpu": props.name, "nvidia_smi": q, "rounds": ROUNDS, "steps_per_round": steps,
                      "kernels": "fast", "results": rows}))


if __name__ == "__main__":
    main()
