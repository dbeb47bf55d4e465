"""adapt() of a distributed multi-level context (cup2d_amr_adapt on cup2d_amr_create_ranks) against the plain context's
(needs a GPU; not part of bench.py's contract line).

  python tools/bench_amr_adapt_ranks.py [base_level ...]                (default: 5 7 9; base 9 is config C5)
  torchrun --nproc-per-node N tools/bench_amr_adapt_ranks.py [base ...]  (N GPUs: the distributed call only, per rank)

On one GPU, for each synthetic three-level mesh of tools/bench_amr_adapt.py (same fields, tolerances and headroom), a plain
cup2d_amr_adapt and a one-rank distributed one alternate on fresh contexts with the same fields; context creation, uploads
and the first tagging's chi-lab table stay outside the timed window.  Reported per mesh: the host time of every call up to a
device synchronise, the device time of the transfer kernels (amr_regrid_*) and of the decision kernels (amr_adapt_*) from a
torch.profiler run of one call of each kind, whether block lists and fields agree bit for bit, and the card's name and power
limit read in the same run.  Under torchrun every rank prints the same for its share (even initial partition)."""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np

from bench_amr_adapt import FIELDS, fields_of, power_limit


def fresh(blocks, h0, f, lmax, rank=None, rb=None, dist=None, device=0):
    """a plain (rank None) or distributed context with the fields and the tagging's chi-lab table built"""
    from cup2d_b200.amr import AmrSimulation
    if rank is None:
        sim, b0, b1 = AmrSimulation(blocks, 1, 1, h0, 1e-4), 0, len(blocks)
    else:
        sim = AmrSimulation.distributed(blocks, 1, 1, h0, 1e-4, rank, rb, dist, device=device)
        b0, b1 = int(rb[rank]), int(rb[rank + 1])
    sim.adapt_tags(1e300, lmax)
    for n, a in f.items():
        sim.upload(n, a[b0:b1])
    return sim


def timed(sim, rtol, ctol, lmax, dist=None):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    sim.adapt(rtol, ctol, lmax, dist=dist)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def kernel_times(sim, rtol, ctol, lmax, dist=None):
    import torch
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        sim.adapt(rtol, ctol, lmax, dist=dist)
        torch.cuda.synchronize()
    out = {"amr_adapt_": 0.0, "amr_regrid_": 0.0}
    for e in prof.events():
        for tag in out:
            if tag in e.name:
                out[tag] += getattr(e, "device_time_total", 0.0) * 1e-6
    return {"decision_device_s": out["amr_adapt_"], "transfer_device_s": out["amr_regrid_"]}


def setup(base):
    from bench_amr import three_level_mesh
    blocks = three_level_mesh(base)
    h0, lmax = 1.0 / 8, base + 4
    f = fields_of(blocks, h0)
    probe = fresh(blocks, h0, f, lmax)
    linf = probe.adapt_tags(1e300, lmax)
    probe.close()
    return blocks, h0, lmax, f, float(np.quantile(linf, 0.9)), float(np.quantile(linf, 0.4))


def bench_one_gpu(base, reps=2):
    import torch
    blocks, h0, lmax, f, rtol, ctol = setup(base)
    rb = np.array([0, len(blocks)], dtype=np.int64)
    times = {"plain": [], "distributed": []}
    same = True
    for r in range(reps + 1):            # the first round warms both paths up and is not reported
        a = fresh(blocks, h0, f, lmax)
        ta = timed(a, rtol, ctol, lmax)
        b = fresh(blocks, h0, f, lmax, 0, rb)
        tb = timed(b, rtol, ctol, lmax)
        if r:
            times["plain"].append(ta)
            times["distributed"].append(tb)
        same &= bool(np.array_equal(a.blocks, b.blocks))
        for n in FIELDS:
            same &= bool(np.array_equal(a.download(n), b.download(n)))
        nnew = len(a.blocks)
        a.close()
        b.close()
    a = fresh(blocks, h0, f, lmax)
    ka = kernel_times(a, rtol, ctol, lmax)
    a.close()
    b = fresh(blocks, h0, f, lmax, 0, rb)
    kb = kernel_times(b, rtol, ctol, lmax)
    b.close()
    print(json.dumps({
        "workload": f"adapt() of the synthetic 3-level mesh, base level {base}", "blocks_old": len(blocks), "blocks_new": nnew,
        "plain_call_s": times["plain"], "distributed_1rank_call_s": times["distributed"], "plain_kernels": ka,
        "distributed_1rank_kernels": kb, "same_blocks_and_fields": same,
        "gpu": torch.cuda.get_device_properties(0).name, "power_limit": power_limit()}), flush=True)
    return same


def bench_ranks(base, reps=2):
    import torch
    import torch.distributed as td
    rank, W = td.get_rank(), td.get_world_size()
    blocks, h0, lmax, f, rtol, ctol = setup(base)
    rb = np.array([len(blocks) * r // W for r in range(W + 1)], dtype=np.int64)
    times = []
    for r in range(reps + 1):
        s = fresh(blocks, h0, f, lmax, rank, rb, td, device=rank)
        t = timed(s, rtol, ctol, lmax, dist=td)
        if r:
            times.append(t)
        new_rb = s.rank_begin().tolist()
        td.barrier()
        s.close()
    s = fresh(blocks, h0, f, lmax, rank, rb, td, device=rank)
    k = kernel_times(s, rtol, ctol, lmax, dist=td)
    td.barrier()
    s.close()
    print(json.dumps({
        "workload": f"distributed adapt() of the synthetic 3-level mesh, base level {base}", "rank": rank, "ranks": W,
        "blocks_old": len(blocks), "rank_begin_old": rb.tolist(), "rank_begin_new": new_rb, "call_s": times, **k,
        "gpu": torch.cuda.get_device_properties(rank).name, "power_limit": power_limit()}), flush=True)
    return True


if __name__ == "__main__":
    bases = [int(x) for x in sys.argv[1:]] or [5, 7, 9]
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        import torch
        import torch.distributed as td
        td.init_process_group("gloo")
        torch.cuda.set_device(td.get_rank())
        ok = all([bench_ranks(b) for b in bases])
        td.destroy_process_group()
    else:
        ok = all([bench_one_gpu(b) for b in bases])
    sys.exit(0 if ok else 1)
