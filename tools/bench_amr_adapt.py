"""adapt() of a multi-level device context, composed against one call (needs a GPU; not part of bench.py's contract line).

  python tools/bench_amr_adapt.py [base_level ...]      (default: 5 7 9; base 9 is config C5, 501 376 blocks)

For each synthetic three-level mesh (tools/bench_amr.py three_level_mesh, seeded fields, tolerances at quantiles of the
device's tags as in `bench_amr.py regrid`), the two paths alternate on fresh contexts with the same fields, context creation,
uploads and the first tagging's host-built chi-lab table outside the timed window:
  - composed: cup2d_amr_adapt_tags (download), cup2d_amr_adapt_mesh (host decision, called twice: size, fill), then
    cup2d_amr_regrid (host classification, new plan, transfer kernels);
  - device:   cup2d_amr_adapt (tags, decision, order and classification on the device, new plan on the host, transfer).
Each is timed with a host clock up to a device synchronise.  Reported per mesh: the times of every repetition, the host
decision alone, the new plan alone (AmrPlan of the new list: the host part both paths keep), a separate torch.profiler run
of cup2d_amr_adapt with the device time of its decision / sort kernels (amr_adapt_*) and transfer kernels (amr_regrid_*),
whether the block lists and all seven fields agree bit for bit, and the card's name and power limit.  One JSON line per mesh."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np

FIELDS = ("vel", "vold", "tmpV", "pres", "pold", "chi", "tmp")


def fields_of(blocks, h0):
    from bench_amr import seeded_fields
    vel, pres = seeded_fields(blocks, h0)
    rng = np.random.default_rng(0)
    vel = vel + 0.05 * rng.uniform(-1, 1, vel.shape)
    return {"vel": vel, "vold": vel, "tmpV": 0 * vel, "pres": pres, "pold": pres, "chi": 0 * pres, "tmp": pres}


def fresh(blocks, h0, f, lmax=None):
    """a context with the fields; with lmax, also the tagging's chi-lab table, which the first tagging on a context builds on
    the host (the same cost on both paths, kept out of the timed window), after which the fields are uploaded again"""
    from cup2d_b200.amr import AmrSimulation
    sim = AmrSimulation(blocks, 1, 1, h0, 1e-4)
    if lmax is not None:
        sim.adapt_tags(1e300, lmax)
    for n, a in f.items():
        sim.upload(n, a)
    return sim


def composed(sim, rtol, ctol, lmax):
    from cup2d_b200.amr import adapt_mesh
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    linf = sim.adapt_tags(rtol, lmax)
    t1 = time.perf_counter()
    new = adapt_mesh(sim.blocks, 1, 1, lmax, linf, rtol, ctol)
    t2 = time.perf_counter()
    sim.regrid(new)
    torch.cuda.synchronize()
    t3 = time.perf_counter()
    return {"total": t3 - t0, "tags": t1 - t0, "decision": t2 - t1, "regrid": t3 - t2}


def device(sim, rtol, ctol, lmax):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    sim.adapt(rtol, ctol, lmax)
    torch.cuda.synchronize()
    return {"total": time.perf_counter() - t0}


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip()
    except Exception:
        return "unknown"


def bench(base, reps=2):
    import torch
    from bench_amr import three_level_mesh
    from cup2d_b200.amr import AmrPlan
    blocks = three_level_mesh(base)
    h0, lmax = 1.0 / 8, base + 4   # one level of headroom: the finest blocks may refine too
    f = fields_of(blocks, h0)
    probe = fresh(blocks, h0, f)
    linf = probe.adapt_tags(1e300, lmax)
    probe.close()
    rtol, ctol = float(np.quantile(linf, 0.9)), float(np.quantile(linf, 0.4))
    times = {"composed": [], "device": []}
    same_blocks = same_fields = True
    new = None
    for r in range(reps + 1):        # the first round warms both paths up and is not reported
        a = fresh(blocks, h0, f, lmax)
        ta = composed(a, rtol, ctol, lmax)
        b = fresh(blocks, h0, f, lmax)
        tb = device(b, rtol, ctol, lmax)
        if r:
            times["composed"].append(ta)
            times["device"].append(tb)
        same_blocks &= bool(np.array_equal(a.blocks, b.blocks))
        for n in FIELDS:
            same_fields &= bool(np.array_equal(a.download(n), b.download(n)))
        new = a.blocks.copy()
        a.close()
        b.close()
    old = {tuple(x): k for k, x in enumerate(blocks.tolist())}
    nref = sum((l - 1, i // 2, j // 2) in old for l, i, j in new.tolist()) // 4
    ncomp = sum((l + 1, 2 * i, 2 * j) in old for l, i, j in new.tolist())
    t0 = time.perf_counter()
    AmrPlan(new, 1, 1).close()
    t_plan = time.perf_counter() - t0
    # device time of the kernels of one cup2d_amr_adapt, in a run of its own
    c = fresh(blocks, h0, f, lmax)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        c.adapt(rtol, ctol, lmax)
        torch.cuda.synchronize()
    c.close()
    dev, launches = {}, {}
    for e in prof.events():
        for tag in ("amr_adapt_", "amr_regrid_"):
            if tag in e.name:
                k = e.name.split("(")[0].split("::")[-1].replace("void ", "")
                dev[k] = dev.get(k, 0.0) + getattr(e, "device_time_total", 0.0) * 1e-6
                launches[k] = launches.get(k, 0) + 1
    t_decision_dev = sum(v for k, v in dev.items() if k.startswith("amr_adapt_"))
    t_transfer_dev = sum(v for k, v in dev.items() if k.startswith("amr_regrid_"))
    print(json.dumps({
        "workload": f"adapt() of the synthetic 3-level mesh, base level {base}", "blocks_old": len(blocks),
        "blocks_new": len(new), "refined": nref, "compressed_groups": ncomp,
        "composed_s": times["composed"], "device_s": [t["total"] for t in times["device"]],
        "speedup_median": float(np.median([t["total"] for t in times["composed"]]) /
                                np.median([t["total"] for t in times["device"]])),
        "new_plan_host_s": t_plan, "decision_sort_device_s": t_decision_dev, "transfer_device_s": t_transfer_dev,
        "per_kernel_s": dev, "launches": launches,
        "same_blocks": same_blocks, "same_fields": same_fields,
        "gpu": torch.cuda.get_device_properties(0).name, "power_limit": power_limit()}), flush=True)
    return same_blocks and same_fields


if __name__ == "__main__":
    bases = [int(x) for x in sys.argv[1:]] or [5, 7, 9]
    ok = all([bench(b) for b in bases])
    sys.exit(0 if ok else 1)
