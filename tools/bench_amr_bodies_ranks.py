"""The body calls on distributed multi-level contexts: cup2d_amr_ongrid, _surface, _forces and _collide of the two Nm-1161-class
fish of tools/bench_amr.py (ongrid / collide / forces: L = 0.05, overlapping, in the finest region of the config C5 mesh) with
seeded vel and pres.

  python tools/bench_amr_bodies_ranks.py [base_level=9] [reps=10]
      one GPU: a plain context (cup2d_amr_create) against a one-rank distributed context (cup2d_amr_create_ranks), the two
      timed alternately in the same process; the results must be bitwise equal
  python -m torch.distributed.run --nproc-per-node N tools/bench_amr_bodies_ranks.py [base_level=9] [reps=10]
      N GPUs of one box: the mesh split into N equal block ranges, every rank times its calls

Each call is timed with CUDA events on the legacy default stream, which the contexts' blocking streams are ordered with, so an
event pair brackets the whole call (uploads, kernels, halo refreshes, the all-reduce, downloads, host work); medians over
`reps` calls after 2 warm-up calls.  One JSON line per process, with the card's name and power limit read in the same run."""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle")]

CALLS = ("ongrid", "surface", "forces", "collide")


def workload(base):
    import amr_body_oracle as bo
    from bench_amr import seeded_fields, three_level_mesh
    blocks = three_level_mesh(base)
    h0 = 1.0 / 8
    hmin = h0 / (1 << int(blocks[:, 0].max()))
    L = 0.05
    nm = 8 * int(np.ceil(L / (hmin / np.sqrt(2)) / 8)) + 1
    bodies = [bo.synthetic_body((0.48, 0.52), L, nm, 0.2), bo.synthetic_body((0.4802, 0.5204), L, nm, 0.25, phase=1.0)]
    vel, pres = seeded_fields(blocks, h0)
    return blocks, h0, L, nm, bodies, vel, pres


def calls(sim, bodies, L):
    """the four calls as closures over `sim`, and a function returning their results (for the equality check)"""
    state = {}

    def ongrid():
        state["out"] = sim.ongrid(bodies)

    def motions():
        out = state["out"]
        return [{"u": 0.1 - 0.2 * k, "v": 0.05 - 0.1 * k, "omega": 0.3 - 0.6 * k, "center_of_mass": out[k, 3:5], "M": out[k, 5],
                 "J": out[k, 6], "length": L} for k in range(2)]

    def forces():
        state["f"] = sim.forces(motions())

    def collide():
        state["c"] = sim.collide(motions())
    fns = {"ongrid": ongrid, "surface": lambda: sim.surface(2), "forces": forces, "collide": collide}
    return fns, lambda: (state["out"], state["f"], state["c"][0], state["c"][1])


def time_call(f):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    f()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


def card():
    import torch
    props = torch.cuda.get_device_properties(torch.cuda.current_device())
    try:
        power = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit", "--format=csv,noheader"],
                               capture_output=True, text=True).stdout.strip()
    except Exception:
        power = "unknown"
    return props.name, power


def one_gpu(base, reps):
    from cup2d_b200.amr import AmrSimulation
    blocks, h0, L, nm, bodies, vel, pres = workload(base)
    nb = len(blocks)
    t0 = time.perf_counter()
    plain = AmrSimulation(blocks, 1, 1, h0, 1e-4)
    t_plain = time.perf_counter() - t0
    t0 = time.perf_counter()
    dist = AmrSimulation.distributed(blocks, 1, 1, h0, 1e-4, 0, [0, nb])
    t_dist = time.perf_counter() - t0
    sims = {"plain": plain, "distributed_1rank": dist}
    fns, results = {}, {}
    for name, sim in sims.items():
        sim.upload("vel", vel)
        sim.upload("pres", pres)
        fns[name], results[name] = calls(sim, bodies, L)
    ms = {name: {c: [] for c in CALLS} for name in sims}
    for rep in range(reps + 2):              # the two forms alternate, call by call
        for c in CALLS:
            for name in sims:
                t = time_call(fns[name][c])
                if rep >= 2:
                    ms[name][c].append(t)
    a, b = results["plain"](), results["distributed_1rank"]()
    same = all(np.array_equal(x, y) for x, y in zip(a, b))
    same = same and all(np.array_equal(plain.shape_get(k)[n], dist.shape_get(k)[n]) for k in range(2) for n in ("ids", "chi", "dist", "udef"))
    nob = [len(plain.shape_get(k, dist=False)["ids"]) for k in range(2)]
    gpu, power = card()
    med = {name: {c: float(np.median(v)) for c, v in d.items()} for name, d in ms.items()}
    print(json.dumps({"workload": f"ongrid + surface + forces + collide of two overlapping fish (Nm {nm}) on the synthetic 3-level mesh, base level {base}",
                      "blocks": nb, "obstacle_blocks": nob, "reps": reps, "ms_median": med,
                      "ms_min": {name: {c: float(np.min(v)) for c, v in d.items()} for name, d in ms.items()},
                      "distributed_over_plain": {c: med["distributed_1rank"][c] / med["plain"][c] for c in CALLS},
                      "create_s": {"plain": t_plain, "distributed_1rank": t_dist}, "bitwise_equal": bool(same),
                      "gpu": gpu, "power_limit": power}))
    plain.close()
    dist.close()
    if not same:
        sys.exit("the one-rank distributed context differs from the plain context")


def ranks(base, reps):
    import torch
    import torch.distributed as td
    from cup2d_b200.amr import AmrSimulation
    td.init_process_group("gloo")
    rank, W = td.get_rank(), td.get_world_size()
    torch.cuda.set_device(rank)
    blocks, h0, L, nm, bodies, vel, pres = workload(base)
    nb = len(blocks)
    rb = [nb * r // W for r in range(W + 1)]
    sim = AmrSimulation.distributed(blocks, 1, 1, h0, 1e-4, rank, rb, td, device=rank)
    sl = slice(rb[rank], rb[rank + 1])
    sim.upload("vel", vel[sl])
    sim.upload("pres", pres[sl])
    fns, _ = calls(sim, bodies, L)
    ms = {c: [] for c in CALLS}
    for rep in range(reps + 2):
        for c in CALLS:
            t = time_call(fns[c])
            if rep >= 2:
                ms[c].append(t)
    gpu, power = card()
    print(json.dumps({"workload": f"the four body calls on {W} ranks, base level {base}", "rank": rank, "blocks": nb,
                      "rank_blocks": rb[rank + 1] - rb[rank], "ms_median": {c: float(np.median(v)) for c, v in ms.items()},
                      "gpu": gpu, "power_limit": power}), flush=True)
    td.barrier()
    sim.close()
    td.destroy_process_group()


if __name__ == "__main__":
    base = int(sys.argv[1]) if len(sys.argv) > 1 else 9
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 10
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        ranks(base, reps)
    else:
        one_gpu(base, reps)
