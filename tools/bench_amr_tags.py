"""adapt()'s tagging on a multi-level device context: the table-gather baseline against the fused kernel of fast contexts (needs
a GPU; not part of bench.py's contract line).

  python tools/bench_amr_tags.py [mesh ...]      (default: runsh 5 6 7 8 9; an integer is the base level of the synthetic
                                                  three-level mesh of tools/bench_amr.py, base 9 being config C5, 501 376
                                                  blocks; runsh is the reference's run.sh mesh of tests/golden/amrtags_lmax8.npz)

Per mesh and mode (baseline: cup2d_amr_set_fast(0); fast: 1), each on a fresh context with the same fields:
  - first_tags_s: wall time of the first cup2d_amr_adapt_tags, its table build included (the baseline builds the full per-cell
    tables of kinds 1 and 3, the fast path the 8-neighbour table and the compact rows of kinds 1 and 3), host clock up to the
    call's own device synchronise;
  - mem_first_tags_bytes: device memory taken by that first call (cudaMemGetInfo before and after);
  - steady_call_s: median host time of one further call (tags + per-block L-inf download);
  - kernel_s: device time per call of the tagging kernels (torch.profiler, CUPTI, over `reps` calls in a run of their own):
    amr_gather_kernel + amr_vorticity_kernel + amr_tag_block_kernel, or amr_tags_fast_kernel;
  - adapt_first_s: one cup2d_amr_adapt on another fresh context, its first tagging inside the window.
Also whether the two modes' L-inf and tagging fields agree bit for bit, and the card's name and power limit.  One JSON line
per mesh."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np

TAG_KERNELS = ("amr_gather_kernel", "amr_vorticity_kernel", "amr_tag_block_kernel", "amr_tags_fast_kernel")


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip()
    except Exception:
        return "unknown"


def case(name):
    """(blocks, bpdx, bpdy, h0, level_max, vel, chi, rtol, ctol)"""
    if name == "runsh":
        d = np.load(os.path.join(ROOT, "tests", "golden", "amrtags_lmax8.npz"))
        return (d["blocks"], int(d["bpdx"]), int(d["bpdy"]), float(d["h0"]), int(d["level_max"]), d["vel"], d["chi"],
                float(d["rtol"]), float(d["ctol"]))
    from bench_amr import seeded_fields, three_level_mesh
    base = int(name)
    blocks = three_level_mesh(base)
    h0 = 1.0 / 8
    vel, _ = seeded_fields(blocks, h0)
    # chi: a disc of body cells in the finest region, so that the chi rule fires there
    rng = np.random.default_rng(base)
    chi = np.zeros((len(blocks), 8, 8, 1))
    fine = np.flatnonzero(blocks[:, 0] == blocks[:, 0].max())
    chi[rng.choice(fine, max(1, len(fine) // 50), replace=False), 3:5, 3:5, 0] = 1.0
    return blocks, 1, 1, h0, base + 4, vel, chi, None, None


def fresh(c, fast):
    from cup2d_b200.amr import AmrSimulation
    blocks, bx, by, h0, _, vel, chi = c[:7]
    sim = AmrSimulation(blocks, bx, by, h0, 1e-4)
    sim.set_fast(fast)
    sim.upload("vel", vel)
    sim.upload("chi", chi)
    return sim


def one_mode(c, fast, rtol, ctol, reps):
    import torch
    lmax = c[4]
    sim = fresh(c, fast)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    t0 = time.perf_counter()
    linf = sim.adapt_tags(rtol, lmax)
    t_first = time.perf_counter() - t0
    mem = free0 - torch.cuda.mem_get_info()[0]
    tmp = sim.download("tmp")
    steady = []
    for _ in range(reps):
        t0 = time.perf_counter()
        sim.adapt_tags(rtol, lmax)
        steady.append(time.perf_counter() - t0)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            sim.adapt_tags(rtol, lmax)
        torch.cuda.synchronize()
    sim.close()
    kern = {}
    for e in prof.events():
        k = e.name.split("(")[0].split("::")[-1].replace("void ", "")
        if k in TAG_KERNELS:
            kern[k] = kern.get(k, 0.0) + getattr(e, "device_time_total", 0.0) * 1e-6 / reps
    a = fresh(c, fast)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    a.adapt(rtol, ctol, lmax)
    torch.cuda.synchronize()
    t_adapt = time.perf_counter() - t0
    nnew = len(a.blocks)
    a.close()
    return dict(first_tags_s=t_first, mem_first_tags_bytes=int(mem), steady_call_s=float(np.median(steady)),
                kernel_s=sum(kern.values()), per_kernel_s=kern, adapt_first_s=t_adapt, blocks_new=nnew), linf, tmp


def bench(name, reps=20):
    import torch
    c = case(name)
    rtol, ctol = c[7], c[8]
    if rtol is None:   # tolerances at quantiles of the tags, as tools/bench_amr_adapt.py
        probe = fresh(c, True)
        linf = probe.adapt_tags(1e300, c[4])
        probe.close()
        rtol, ctol = float(np.quantile(linf, 0.9)), float(np.quantile(linf, 0.4))
    out = {"workload": f"adapt()'s tagging, mesh {name}", "blocks": len(c[0]), "level_max": c[4]}
    res = {}
    for mode, fast in (("fast", True), ("baseline", False)):
        out[mode], *res[mode] = one_mode(c, fast, rtol, ctol, reps)
    out["bitwise_equal"] = bool(np.array_equal(res["fast"][0].view(np.uint64), res["baseline"][0].view(np.uint64)) and
                                np.array_equal(res["fast"][1].view(np.uint64), res["baseline"][1].view(np.uint64)))
    out["gpu"], out["power_limit"] = torch.cuda.get_device_properties(0).name, power_limit()
    print(json.dumps(out), flush=True)
    return out["bitwise_equal"]


if __name__ == "__main__":
    import torch
    torch.cuda.init()
    names = sys.argv[1:] or ["runsh", "5", "6", "7", "8", "9"]
    ok = all([bench(n) for n in names])
    sys.exit(0 if ok else 1)
