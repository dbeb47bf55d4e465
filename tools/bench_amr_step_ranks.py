"""Needs a GPU (not part of bench.py's line): wall time per multi-level step on DISTRIBUTED contexts (cup2d_amr_create_ranks),
the blocking cup2d_amr_step against the enqueued form (cup2d_amr_step_enqueue + cup2d_amr_step_result, replayed as a CUDA
graph), and on one rank also the plain context's (cup2d_amr_create) enqueued step, so that the cost of the distributed
path itself is visible.  Synthetic three-level meshes of tools/bench_amr.py at base levels 5-9 (9 = config C5), fast
kernels, 10 fixed Krylov iterations and a tolerance-driven solve (tol_abs 1e-7, at most 100 iterations).  The forms
alternate over ROUNDS rounds in this one process, every timed step ends in a device synchronise, all are warmed up first.
  python tools/bench_amr_step_ranks.py [max_base_level=9] [steps_per_round=10]                  one GPU, one rank
  torchrun --nproc_per_node=N tools/bench_amr_step_ranks.py [max_base_level] [steps_per_round]    N GPUs, N ranks
Rank 0 prints one JSON line with the card's name and power limit (median and 10th-90th percentile per step, in ms; on
several ranks the slowest rank's time of each step)."""
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


def bench_mesh(label, blocks, h0, nu, vel, pres, steps, rank, world, td):
    import torch
    from cup2d_b200.amr import AmrSimulation
    nb = len(blocks)
    rb = np.array([nb * r // world for r in range(world + 1)], dtype=np.int64)
    b0, b1 = int(rb[rank]), int(rb[rank + 1])
    out = {"mesh": label, "blocks": int(nb), "levels": sorted(set(blocks[:, 0].tolist())), "rank_begin": rb.tolist()}
    forms = ("blocking", "enqueued") + (("plain_enqueued",) if world == 1 else ())
    sims = {}                        # one context per form (a distributed context's host set-up is seconds at C5)
    for form in forms:
        if form == "plain_enqueued":
            sims[form] = AmrSimulation(blocks, 1, 1, h0, nu)
            sims[form].set_fast(True)
        else:
            sims[form] = AmrSimulation.distributed(blocks, 1, 1, h0, nu, rank, rb, td, device=torch.cuda.current_device())
    for sname, kw in SOLVES.items():
        for s in sims.values():      # every solve column starts from the same fields
            s.upload("vel", vel[b0:b1])
            s.upload("pres", pres[b0:b1])

        def one(form):
            s = sims[form]
            if form == "blocking":
                r = s.step(cfl=0.5, **kw)
            else:
                s.step_enqueue(cfl=0.5, **kw)
                r = s.step_result()
            torch.cuda.synchronize()
            return r

        for form in forms:           # warm-up: tables, the direct first enqueue and the graph capture
            for _ in range(3):
                one(form)
        wall = {f: [] for f in forms}
        iters = {f: [] for f in forms}
        for _ in range(ROUNDS):
            for form in forms:
                if td is not None:
                    td.barrier()
                for _ in range(steps):
                    t0 = time.perf_counter()
                    r = one(form)
                    wall[form].append((time.perf_counter() - t0) * 1e3)
                    iters[form].append(r[1])
        if td is not None:           # per step, the slowest rank
            for form in forms:
                allw = [None] * world
                td.all_gather_object(allw, wall[form])
                wall[form] = np.max(np.asarray(allw), axis=0).tolist()
        res = {f: median_spread(wall[f]) | {"iters_median": float(np.median(iters[f]))} for f in forms}
        res["speedup_enqueued_over_blocking"] = res["blocking"]["median"] / res["enqueued"]["median"]
        if "plain_enqueued" in res:
            res["distributed_over_plain_enqueued"] = res["enqueued"]["median"] / res["plain_enqueued"]["median"]
        out[sname] = res
    if td is not None:
        td.barrier()                 # no rank frees its arrays while a peer may still read them
    for s in sims.values():
        s.close()
    return out


def main():
    import torch
    import bench_amr
    maxb = int(sys.argv[1]) if len(sys.argv) > 1 else 9
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 10
    td, rank, world = None, 0, 1
    if "WORLD_SIZE" in os.environ and int(os.environ["WORLD_SIZE"]) > 1:
        import torch.distributed as td
        td.init_process_group("gloo")
        rank, world = td.get_rank(), td.get_world_size()
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
    props = torch.cuda.get_device_properties(torch.cuda.current_device())
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    rows = []
    for base in range(5, maxb + 1):
        blocks = bench_amr.three_level_mesh(base)
        h0 = 1.0 / 8
        vel, pres = bench_amr.seeded_fields(blocks, h0)
        rows.append(bench_mesh(f"synthetic base {base}" + (" (C5)" if base == 9 else ""), blocks, h0, 1e-4, vel, pres, steps,
                               rank, world, td))
        if rank == 0:
            print(f"# {rows[-1]['mesh']}: " + ", ".join(f"{s} {f} {rows[-1][s][f]['median']:.3f} ms" for s in SOLVES
                                                       for f in rows[-1][s] if isinstance(rows[-1][s][f], dict)), flush=True)
    if rank == 0:
        print(json.dumps({"tool": "bench_amr_step_ranks", "gpu": props.name, "nvidia_smi": q, "ranks": world, "rounds": ROUNDS,
                          "steps_per_round": steps, "kernels": "fast", "results": rows}))
    if td is not None:
        td.destroy_process_group()


if __name__ == "__main__":
    main()
