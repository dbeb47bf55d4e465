"""Round-2 tool (needs a GPU; not part of bench.py's contract line): multi-level time steps on the mesh the unmodified
reference grows for its run.sh case (config C5 of SURVEY 8(d) at the chosen levelMax).

  python tools/bench_amr.py [levelMax=9] [steps=10] [poisson_iters=10] [fast=1]
  python tools/bench_amr.py synthetic [base_level=9] [steps=10] [poisson_iters=10] [fast=1]     (config C5: 3 levels;
      under torchrun on N GPUs: the mesh distributed by block ranges, cup2d_amr_create_ranks)
  python tools/bench_amr.py regrid [base_level=9]      one adapt() of the C5 mesh: decision, regrid, transfer kernels
  python tools/bench_amr.py ongrid [base_level=9]      cup2d_amr_ongrid of two fish in the finest region of the C5 mesh
  python tools/bench_amr.py collide [base_level=9]     cup2d_amr_collide of two overlapping fish there, after ongrid
  python tools/bench_amr.py forces [base_level=9]      cup2d_amr_surface + cup2d_amr_forces of the same two fish, seeded vel, pres

The mesh comes from oracle/_ref/ref_harness amrlab (which travels to the GPU box prebuilt), the fields are its seeded ones,
bodies are left out (u_def = 0, chi = 0).  Prints one JSON line: blocks, cells, levels, ms per step with CUDA events on the
context's stream, Mcell-updates/s = cells * (2 + K) / time, and the host-side plan build time."""
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np


def three_level_mesh(base_level, r1=0.22, r2=0.11, centre=(0.5, 0.5)):
    """Synthetic 3-level mesh for config C5 (SURVEY 8(d): 3-level block-AMR, 16384^2 effective resolution at base_level 9):
    a unit square of 2^base_level blocks per side; the base blocks within r2 of `centre` are refined twice, those within r1
    (and, for the 2:1 rule, every 8-neighbour of a twice-refined one) once.  Refinement is uniform inside a base block, so level
    jumps occur between base blocks only and never exceed one.  Blocks follow the library's space-filling-curve order of the
    base blocks, children in Z order.  Returns int32 (level, i, j) triples."""
    from cup2d_b200 import lib as _l
    import ctypes as C
    n = 1 << base_level
    ij = np.empty(2 * n * n, dtype=np.int32)
    _l.check(_l.load_library().cup2d_block_order(1, 1, base_level, ij.ctypes.data_as(C.POINTER(C.c_int32))))
    ij = ij.reshape(-1, 2)
    x, y = (ij[:, 0] + 0.5) / n - centre[0], (ij[:, 1] + 0.5) / n - centre[1]
    d2 = x * x + y * y
    depth = np.zeros((n, n), dtype=np.int32)          # [j, i]
    depth[ij[:, 1], ij[:, 0]] = (d2 < r1 * r1).astype(np.int32) + (d2 < r2 * r2)
    two = np.pad(depth == 2, 1)
    near_two = np.zeros_like(depth, dtype=bool)
    for dj in range(3):
        for di in range(3):
            near_two |= two[dj:dj + n, di:di + n]
    depth = np.maximum(depth, near_two.astype(np.int32))
    dep = depth[ij[:, 1], ij[:, 0]]
    out = []
    for d in range(3):
        sel = ij[dep == d]
        m = 1 << d
        cj, ci = np.meshgrid(np.arange(m), np.arange(m), indexing="ij")     # Z order would interleave; row-major is fine for d <= 2
        t = np.empty((len(sel), m * m, 3), dtype=np.int32)
        t[:, :, 0] = base_level + d
        t[:, :, 1] = sel[:, 0:1] * m + ci.reshape(1, -1)
        t[:, :, 2] = sel[:, 1:2] * m + cj.reshape(1, -1)
        out.append((np.flatnonzero(dep == d), t))
    # stitch back in curve order of the base blocks
    counts = np.array([1, 4, 16])[dep]
    start = np.concatenate([[0], np.cumsum(counts)])
    blocks = np.empty((start[-1], 3), dtype=np.int32)
    for d, (pos, t) in enumerate(out):
        m2 = 1 << (2 * d)
        idx = (start[pos][:, None] + np.arange(m2)[None, :]).reshape(-1)
        blocks[idx] = t.reshape(-1, 3)
    return blocks


def seeded_fields(blocks, h0):
    """Taylor-Green velocity + a smooth pressure on the cell centres of a multi-level mesh"""
    h = h0 / (1 << blocks[:, 0]).astype(np.float64)
    ix = np.arange(8, dtype=np.float64) + 0.5
    X = (blocks[:, 1] * 8)[:, None, None] * h[:, None, None] + h[:, None, None] * ix[None, None, :] + 0 * ix[None, :, None]
    Y = (blocks[:, 2] * 8)[:, None, None] * h[:, None, None] + h[:, None, None] * ix[None, :, None] + 0 * ix[None, None, :]
    vel = np.stack([np.sin(2 * np.pi * X) * np.cos(2 * np.pi * Y), -np.cos(2 * np.pi * X) * np.sin(2 * np.pi * Y)], axis=-1)
    pres = (np.cos(2 * np.pi * X) * np.cos(2 * np.pi * Y))[..., None]
    return vel, pres


def run(sim, nb, blocks, steps, K, label, t_create, fast):
    import torch
    for _ in range(3):
        sim.step(cfl=0.5, max_iter=K)
    torch.cuda.synchronize()
    t0 = time.time()
    for _ in range(steps):
        sim.step(cfl=0.5, max_iter=K)
    torch.cuda.synchronize()
    wall = (time.time() - t0) / steps
    cells = nb * 64
    levels = sorted(set(blocks[:, 0].tolist()))
    print(json.dumps({"workload": label, "blocks": nb, "cells": cells, "levels": levels,
                      "fast": bool(fast), "poisson_iters": K, "ms_per_step_wall": wall * 1e3,
                      "Mcell_updates_per_s": cells * (2 + K) / wall / 1e6, "create_s": t_create}))


def regrid(base):
    """one adapt() of the C5 synthetic mesh with seeded fields, tolerances at quantiles of the device's tagging field so that a
    sizeable share of the blocks refines and of the groups compresses: host time of the decision (cup2d_amr_adapt_mesh), wall
    time of cup2d_amr_regrid, device time of its transfer kernels (torch.profiler), their bytes per new cell against the
    algorithmic figure (each of the six transferred fields read once and written once: 2 x 8 doubles = 128 B per cell, plus
    the lab gather of the refined parents)"""
    import torch
    from cup2d_b200.amr import AmrSimulation, adapt_mesh
    blocks = three_level_mesh(base)
    h0, lmax = 1.0 / 8, base + 4   # one level of headroom: the finest blocks may refine too
    vel, pres = seeded_fields(blocks, h0)
    rng = np.random.default_rng(0)
    vel = vel + 0.05 * rng.uniform(-1, 1, vel.shape)
    sim = AmrSimulation(blocks, 1, 1, h0, 1e-4)
    for n, a in (("vel", vel), ("vold", vel), ("pres", pres), ("pold", pres), ("tmp", pres)):
        sim.upload(n, a)
    linf = sim.adapt_tags(1e300, lmax)
    rtol, ctol = float(np.quantile(linf, 0.9)), float(np.quantile(linf, 0.4))
    t0 = time.perf_counter()
    new = adapt_mesh(blocks, 1, 1, lmax, linf, rtol, ctol)
    t_decision = time.perf_counter() - t0
    old = {tuple(b): k for k, b in enumerate(blocks.tolist())}
    nref = sum((l - 1, i // 2, j // 2) in old for l, i, j in new.tolist()) // 4
    ncomp = sum((l + 1, 2 * i, 2 * j) in old for l, i, j in new.tolist())
    from cup2d_b200.amr import AmrPlan
    t0 = time.perf_counter()
    AmrPlan(new, 1, 1).close()
    t_plan = time.perf_counter() - t0
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        t0 = time.perf_counter()
        sim.regrid(new)
        t_wall = time.perf_counter() - t0
        torch.cuda.synchronize()
    dev = {}
    for e in prof.events():
        if e.name.startswith("amr_regrid_") or "amr_regrid_" in e.name:
            k = e.name.split("(")[0].split("::")[-1].replace("void ", "")
            dev[k] = dev.get(k, 0.0) + getattr(e, "device_time_total", 0.0) * 1e-6
    t_dev = sum(dev.values())
    cells = len(new) * 64
    algo = 128 * cells + nref * (100 * 2 * 2 + 100 * 4) * 8   # + the parents' labs (2 vector + 4 scalar fields), read and written
    props = torch.cuda.get_device_properties(0)
    try:
        import subprocess as sp
        power = sp.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except Exception:
        power = "unknown"
    print(json.dumps({"workload": f"regrid of the synthetic 3-level mesh, base level {base}", "blocks_old": len(blocks),
                      "blocks_new": len(new), "refined": nref, "compressed_groups": ncomp, "t_decision_s": t_decision,
                      "t_new_plan_s": t_plan, "t_regrid_wall_s": t_wall, "t_host_part_s": t_wall - t_dev,
                      "t_transfer_device_s": t_dev, "per_kernel_s": dev,
                      "bytes_per_cell_algorithmic": algo / cells, "GB_per_s_algorithmic": algo / t_dev / 1e9 if t_dev else None,
                      "gpu": props.name, "power_limit": power}))
    sim.close()


def ongrid(base, reps=20):
    """cup2d_amr_ongrid of two run.sh-sized fish (L = 0.2 at the C5 scale: 0.2 / 4 of the unit square, Nm of the reference at
    that resolution) inside the finest region of the C5 mesh, after warm-up: the whole call and each kernel class timed with CUDA
    events on the context's stream (cup2d_amr_ongrid_timing; median over the calls), the host wall time per call, the
    reset/scan kernel against its algorithmic bytes (16 B per cell + the block tables it reads: (i, j), h, the mask it writes),
    and the PCIe bytes per step the call replaces (chi field upload 8 B/cell + the obstacle blocks)"""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import amr_body_oracle as bo
    from cup2d_b200.amr import AmrSimulation
    blocks = three_level_mesh(base)
    h0 = 1.0 / 8
    hmin = h0 / (1 << int(blocks[:, 0].max()))
    L = 0.05
    nm = 8 * int(np.ceil(L / (hmin / np.sqrt(2)) / 8)) + 1   # about the reference's midline spacing, minH / sqrt(2)
    bodies = [bo.synthetic_body((0.48, 0.52), L, nm, 0.2), bo.synthetic_body((0.53, 0.50), L, nm, 3.0, phase=1.0)]
    sim = AmrSimulation(blocks, 1, 1, h0, 1e-4)
    for _ in range(3):
        out = sim.ongrid(bodies)
    t0 = time.perf_counter()
    for _ in range(reps):
        sim.ongrid(bodies)          # returns after its last stream synchronisation
    t_wall = (time.perf_counter() - t0) / reps
    sim.ongrid_timing(True)
    times = []
    for _ in range(reps):
        sim.ongrid(bodies)
        times.append(sim.ongrid_times())
    sim.ongrid_timing(False)
    ms = {k: float(np.median([t[k] for t in times])) for k in sim.ONGRID_TIMES}
    nb = len(blocks)
    nob = [len(sim.shape_get(k, dist=False)["ids"]) for k in range(2)]
    scan_bytes = nb * (64 * 16 + 8 + 8 + 8)
    scan_s = ms["scan"] * 1e-3
    import torch
    props = torch.cuda.get_device_properties(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                               text=True).stdout.strip()
    except Exception:
        power = "unknown"
    print(json.dumps({"workload": f"ongrid of two fish (Nm {nm}) on the synthetic 3-level mesh, base level {base}", "blocks": nb,
                      "obstacle_blocks": nob, "t_call_events_ms": ms["call"], "t_call_wall_ms": t_wall * 1e3,
                      "per_kernel_events_ms": {k: v for k, v in ms.items() if k != "call"},
                      "t_kernels_ms": sum(v for k, v in ms.items() if k != "call"),
                      "scan_bytes_algorithmic": scan_bytes, "scan_GB_per_s": scan_bytes / scan_s / 1e9 if scan_s else None,
                      "pcie_bytes_removed_per_step": nb * 64 * 8 + sum(nob) * (4 + 64 * 8 + 128 * 8),
                      "host_ongrid_time": "not measured at this size", "out": out.tolist(),
                      "gpu": props.name, "power_limit": power}))
    sim.close()


def collide(base, reps=20):
    """cup2d_amr_collide of two run.sh-sized fish (as in ongrid above) placed to overlap along most of their length in the
    finest region of the C5 mesh, after ongrid: the call timed with CUDA events (median over the calls; recorded on the
    legacy default stream, which the context's blocking stream is ordered with, so they bracket the upload, both kernels, the
    download and the host's pair loop), the host wall time per call, and the PCIe bytes per step the call removes (every
    shape's ids, chi, dist and u_def that a host collision model would download)"""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import torch
    import amr_body_oracle as bo
    from cup2d_b200.amr import AmrSimulation
    blocks = three_level_mesh(base)
    h0 = 1.0 / 8
    hmin = h0 / (1 << int(blocks[:, 0].max()))
    L = 0.05
    nm = 8 * int(np.ceil(L / (hmin / np.sqrt(2)) / 8)) + 1
    bodies = [bo.synthetic_body((0.48, 0.52), L, nm, 0.2), bo.synthetic_body((0.4802, 0.5204), L, nm, 0.25, phase=1.0)]
    sim = AmrSimulation(blocks, 1, 1, h0, 1e-4)
    out = sim.ongrid(bodies)
    motions = [{"u": 0.1 - 0.2 * k, "v": 0.05 - 0.1 * k, "omega": 0.3 - 0.6 * k, "center_of_mass": out[k, 3:5], "M": out[k, 5],
                "J": out[k, 6], "length": L} for k in range(2)]
    for _ in range(3):
        uvw, sums = sim.collide(motions)
    t0 = time.perf_counter()
    for _ in range(reps):
        sim.collide(motions)
    t_wall = (time.perf_counter() - t0) / reps
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        sim.collide(motions)
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    ids = [sim.shape_get(k, dist=False)["ids"] for k in range(2)]
    nob = [len(i) for i in ids]
    props = torch.cuda.get_device_properties(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                               text=True).stdout.strip()
    except Exception:
        power = "unknown"
    print(json.dumps({"workload": f"collide of two overlapping fish (Nm {nm}) on the synthetic 3-level mesh, base level {base}",
                      "blocks": len(blocks), "obstacle_blocks": nob, "common_blocks": len(np.intersect1d(*ids)),
                      "iM": sums[:, 0].tolist(), "t_call_events_ms_median": float(np.median(ms)),
                      "t_call_events_ms_min": float(np.min(ms)), "t_call_wall_ms": t_wall * 1e3,
                      "pcie_bytes_removed_per_step": sum(nob) * (4 + 64 * 8 + 64 * 8 + 128 * 8),
                      "uvw_after": uvw.tolist(), "gpu": props.name, "power_limit": power}))
    sim.close()


def forces(base, reps=20):
    """cup2d_amr_surface and cup2d_amr_forces of the two fish of `collide` above, after ongrid, with seeded vel and pres: each
    call timed with CUDA events (median over the calls; recorded on the legacy default stream, which the context's blocking
    stream is ordered with), the host wall time per call, the surface points and obstacle blocks, and the PCIe bytes per step
    the calls remove (vel, pres and chi that host force diagnostics would download: 32 B per cell)"""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import torch
    import amr_body_oracle as bo
    from cup2d_b200.amr import AmrSimulation
    blocks = three_level_mesh(base)
    h0 = 1.0 / 8
    hmin = h0 / (1 << int(blocks[:, 0].max()))
    L = 0.05
    nm = 8 * int(np.ceil(L / (hmin / np.sqrt(2)) / 8)) + 1
    bodies = [bo.synthetic_body((0.48, 0.52), L, nm, 0.2), bo.synthetic_body((0.4802, 0.5204), L, nm, 0.25, phase=1.0)]
    sim = AmrSimulation(blocks, 1, 1, h0, 1e-4)
    out = sim.ongrid(bodies)
    vel, pres = seeded_fields(blocks, h0)
    sim.upload("vel", vel)
    sim.upload("pres", pres)
    motions = [{"u": 0.1 - 0.2 * k, "v": 0.05 - 0.1 * k, "center_of_mass": out[k, 3:5]} for k in range(2)]

    def timed(f):
        for _ in range(3):
            f()
        t0 = time.perf_counter()
        for _ in range(reps):
            f()
        t_wall = (time.perf_counter() - t0) / reps
        ms = []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f()
            e1.record()
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
        return float(np.median(ms)), t_wall * 1e3
    ms_s, wall_s = timed(lambda: sim.surface(2))
    ms_f, wall_f = timed(lambda: sim.forces(motions))
    res = sim.forces(motions)
    npts = [len(sim.surface_get(k)["block"]) for k in range(2)]
    nob = [len(sim.shape_get(k, dist=False)["ids"]) for k in range(2)]
    props = torch.cuda.get_device_properties(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                               text=True).stdout.strip()
    except Exception:
        power = "unknown"
    print(json.dumps({"workload": f"surface + forces of two overlapping fish (Nm {nm}) on the synthetic 3-level mesh, base level {base}",
                      "blocks": len(blocks), "obstacle_blocks": nob, "surface_points": npts,
                      "t_surface_events_ms_median": ms_s, "t_surface_wall_ms": wall_s,
                      "t_forces_events_ms_median": ms_f, "t_forces_wall_ms": wall_f,
                      "pcie_bytes_removed_per_step": len(blocks) * 64 * 32, "forcex": res[:, 2].tolist(), "forcey": res[:, 12].tolist(),
                      "gpu": props.name, "power_limit": power}))
    sim.close()


def main():
    if len(sys.argv) > 1 and sys.argv[1] == "forces":      # python tools/bench_amr.py forces [base_level=9]
        forces(int(sys.argv[2]) if len(sys.argv) > 2 else 9)
        return
    if len(sys.argv) > 1 and sys.argv[1] == "collide":     # python tools/bench_amr.py collide [base_level=9]
        collide(int(sys.argv[2]) if len(sys.argv) > 2 else 9)
        return
    if len(sys.argv) > 1 and sys.argv[1] == "ongrid":      # python tools/bench_amr.py ongrid [base_level=9]
        ongrid(int(sys.argv[2]) if len(sys.argv) > 2 else 9)
        return
    if len(sys.argv) > 1 and sys.argv[1] == "regrid":      # python tools/bench_amr.py regrid [base_level=9]
        regrid(int(sys.argv[2]) if len(sys.argv) > 2 else 9)
        return
    if len(sys.argv) > 1 and sys.argv[1] == "synthetic":   # python tools/bench_amr.py synthetic [base_level=9] [steps] [K] [fast]
        base = int(sys.argv[2]) if len(sys.argv) > 2 else 9
        steps = int(sys.argv[3]) if len(sys.argv) > 3 else 10
        K = int(sys.argv[4]) if len(sys.argv) > 4 else 10
        fast = int(sys.argv[5]) if len(sys.argv) > 5 else 1
        from cup2d_b200.amr import AmrSimulation
        blocks = three_level_mesh(base)
        h0 = 1.0 / 8
        vel, pres = seeded_fields(blocks, h0)
        world, rank, lrank = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))
        t0 = time.time()
        if world > 1:   # under torchrun: the mesh distributed over the GPUs by block ranges (cup2d_amr_create_ranks)
            import torch
            import torch.distributed as dist
            torch.cuda.set_device(lrank)
            dist.init_process_group("nccl", device_id=torch.device("cuda", lrank))
            rb = [round(r * len(blocks) / world) for r in range(world + 1)]
            sim = AmrSimulation.distributed(blocks, 1, 1, h0, 1e-4, rank, rb, dist, device=lrank)
            vel, pres = vel[rb[rank]:rb[rank + 1]], pres[rb[rank]:rb[rank + 1]]
        else:
            sim = AmrSimulation(blocks, 1, 1, h0, 1e-4, device=lrank)
            sim.set_fast(bool(fast))
        sim.upload("vel", vel)
        sim.upload("pres", pres)
        sim.step(cfl=0.5, max_iter=1)          # first step builds the compact tables and the Poisson rows
        t_create = time.time() - t0
        label = f"synthetic 3-level mesh, base level {base} ({8 << (base + 2)}^2 effective), {world} GPU(s)"
        if rank == 0:
            run(sim, len(blocks), blocks, steps, K, label, t_create, fast)
        else:           # same calls, no report (every step synchronises the ranks inside the solve)
            for _ in range(3 + steps):
                sim.step(cfl=0.5, max_iter=K)
        if world > 1:
            dist.barrier()
            dist.destroy_process_group()
        sim.close()
        return
    lmax = int(sys.argv[1]) if len(sys.argv) > 1 else 9
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 10
    K = int(sys.argv[3]) if len(sys.argv) > 3 else 10
    fast = int(sys.argv[4]) if len(sys.argv) > 4 else 1
    import torch
    from cup2d_b200.amr import AmrSimulation
    with tempfile.TemporaryDirectory() as tmp:
        out = os.path.join(tmp, "amr.bin")
        subprocess.run([os.path.join(ROOT, "oracle", "_ref", "ref_harness"), "amrlab", str(lmax), "3", out], check=True,
                       stderr=subprocess.DEVNULL, stdout=subprocess.DEVNULL, env=dict(os.environ, OMP_NUM_THREADS="8"))
        a = np.fromfile(out)
    i, rec = 0, {}
    while i < len(a):
        tag, n = int(a[i]), int(a[i + 1])
        rec[tag] = a[i + 2:i + 2 + n]
        i += 2 + n
    nu, _, h0, bpdx, bpdy, _ = rec[10]
    blocks = rec[11].reshape(-1, 3).astype(np.int32)
    nb = len(blocks)
    t0 = time.time()
    sim = AmrSimulation(blocks, int(bpdx), int(bpdy), h0, nu)
    t_create = time.time() - t0
    sim.upload("vel", rec[12].reshape(nb, 8, 8, 2))
    sim.upload("pres", rec[13].reshape(nb, 8, 8, 1))
    sim.set_fast(bool(fast))
    run(sim, nb, blocks, steps, K, f"run.sh mesh, levelMax {lmax}", t_create, fast)
    sim.close()


if __name__ == "__main__":
    main()
