"""adapt() and regrid on distributed multi-level contexts (cup2d_amr_adapt / cup2d_amr_regrid on cup2d_amr_create_ranks
contexts) against the same call on a plain cup2d_amr_create context with the same fields.  Shared by
tests/test_amr_adapt_ranks_emulation.py (ranks as threads of one process, on the emulated library) and
tests/test_gpu_amr_adapt_ranks.py (one H100: a one-rank distributed context; several GPUs: run as a script under
torch.distributed.run, one process per GPU).

What is compared: the whole new list on every rank; the new partition against rule() below; every rank's tmp, chi, vel,
vold, pres and pold bit for bit with its range of the plain context's fields, tmpV zero; then a few steps on both, to 5e-15
of the largest |value| of each field (bitwise with one rank)."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE, os.path.join(ROOT, "tools"), os.path.join(HERE, "golden")):
    if p not in sys.path:
        sys.path.insert(0, p)

from amr_bodies_ranks import on_threads  # noqa: E402,F401  (re-exported for the tests)

NU = 4e-5
MOVED = ("tmp", "chi", "vel", "vold", "pres", "pold")
FIELDS = MOVED + ("tmpV",)
STEP_TOL = 1e-14


# ---- the reference's new partition, restated -------------------------------------------------------------------------------
def ctrunc(a, b):
    """C integer division: truncates toward zero (Python's // floors)"""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b > 0) else -q


def rule(n):
    """rank_begin of the new partition from n[r] = the new blocks rank r produces (main.cpp:4925-4950 count them as
    blocks_after).  main.cpp:5196-5205: if max / min > 1.01 or min == 0, every rank gets total // W and the first total % W
    one more.  main.cpp:5332-5349 otherwise: flux (n_r - n_{r+1}) / 4 from rank r to r+1, C division, a negative flux
    the other way; rank r keeps n_r - flux_left - flux_right."""
    n = [int(v) for v in n]
    W, total = len(n), sum(n)
    if min(n) == 0 or max(n) / min(n) > 1.01:
        cnt = [total // W + (1 if r < total % W else 0) for r in range(W)]
    else:
        cnt = [n[r] - (ctrunc(n[r] - n[r - 1], 4) if r > 0 else 0) - (ctrunc(n[r] - n[r + 1], 4) if r < W - 1 else 0)
               for r in range(W)]
    return np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)


def full_branch(n):
    return min(n) == 0 or max(n) / min(n) > 1.01


def classify(old, new):
    """(copies {new: old}, children {new: parent}, groups {new: [old ids, J*2 + I order]}) of the step old -> new"""
    at = {tuple(b): k for k, b in enumerate(np.asarray(old).tolist())}
    copies, children, groups = {}, {}, {}
    for q, (l, i, j) in enumerate(np.asarray(new).tolist()):
        if (l, i, j) in at:
            copies[q] = at[(l, i, j)]
        elif (l - 1, i // 2, j // 2) in at:
            children[q] = at[(l - 1, i // 2, j // 2)]
        else:
            groups[q] = [at[(l + 1, 2 * i + a, 2 * j + b)] for b in (0, 1) for a in (0, 1)]
    return copies, children, groups


def owner(rb, g):
    return int(np.searchsorted(rb, g, side="right") - 1)


def produced(old, new, orb):
    """n[r]: new blocks produced by old rank r (a copy or a child on the old block's rank, a compressed parent on the rank of
    its even-i, even-j sibling)"""
    copies, children, groups = classify(old, new)
    n = [0] * (len(orb) - 1)
    for src in list(copies.values()) + list(children.values()) + [g[0] for g in groups.values()]:
        n[owner(orb, src)] += 1
    return n


def properties(old, new, orb, nrb, bpdx, bpdy):
    """what a partition exercises (see test_amr_adapt_ranks_emulation.py)"""
    from cup2d_b200.amr import AmrPlan
    copies, children, groups = classify(old, new)
    n = produced(old, new, orb)
    W = len(orb) - 1
    prop = dict(split_children=False, third_rank_lab=False, group_base_left=False, group_base_right=False,
                producer_empty=min(n) == 0, full=full_branch(n) and W > 1, flux_both=False)
    kids_of = {}
    for q, p in children.items():
        kids_of.setdefault(p, []).append(q)
    if kids_of:
        plan = AmrPlan(old, bpdx, bpdy)
        rp, sb, _, _ = plan.stencil(5)
        plan.close()
    for p, qs in kids_of.items():
        ranks = {owner(nrb, q) for q in qs}
        prop["split_children"] |= len(ranks) > 1
        srcs = {owner(orb, s) for s in sb[rp[p * 100]:rp[(p + 1) * 100]]}
        prop["third_rank_lab"] |= any(len(srcs - {owner(orb, p), r}) > 0 and r != owner(orb, p) for r in ranks)
    for g in groups.values():
        base, others = owner(orb, g[0]), {owner(orb, s) for s in g[1:]}
        if others - {base}:
            prop["group_base_left"] |= any(o > base for o in others)
            prop["group_base_right"] |= any(o < base for o in others)
    if W > 2 and not full_branch(n):
        flux = [ctrunc(n[r] - n[r + 1], 4) for r in range(W - 1)]
        prop["flux_both"] = any(f > 0 for f in flux) and any(f < 0 for f in flux)
    return prop


# ---- cases -------------------------------------------------------------------------------------------------------------------
def seeded_fields(nb, seed):
    rng = np.random.default_rng(seed)
    v = lambda: rng.uniform(-1, 1, (nb, 8, 8, 2))
    s = lambda: rng.uniform(-1, 1, (nb, 8, 8, 1))
    return {"vel": v(), "vold": v(), "tmpV": v(), "pres": s(), "pold": s(), "chi": rng.uniform(0, 1, (nb, 8, 8, 1)), "tmp": s()}


def group_tags(blocks, seed):
    rng = np.random.default_rng(seed)
    groups = {}
    for l, i, j in np.asarray(blocks).tolist():
        groups.setdefault((l, i // 2, j // 2), rng.uniform(0, 1))
    return np.array([groups[(l, i // 2, j // 2)] for l, i, j in np.asarray(blocks).tolist()])


def case(name):
    """dict(blocks, bpdx, bpdy, h0, level_max, rtol, ctol, linf (None: device tags), fields)"""
    if name.startswith("runsh"):      # the run.sh mesh, 278 -> 329 blocks, refinement only
        import make_regrid_golden
        g = make_regrid_golden.load(os.path.join(HERE, "golden", "amrregrid_lmax8.npz"))
        f = seeded_fields(len(g["blocks"]), 7)
        f.update({n: g[n] for n in ("vel", "vold", "pres", "pold", "chi")})
        return dict(blocks=g["blocks"].astype(np.int32), bpdx=int(g["bpdx"]), bpdy=int(g["bpdy"]), h0=float(g["h0"]),
                    level_max=int(g["level_max"]), rtol=float(g["rtol"]), ctol=float(g["ctol"]),
                    linf=None if name == "runsh_device_tags" else g["block_linf"], fields=f)
    if name == "three_level":         # per-group tags: whole groups compress, others refine
        import amr_meshes as M
        import bench_amr
        b = M.reference_order(bench_amr.three_level_mesh(3, r1=0.3, r2=0.15, centre=(0.45, 0.55)), 1, 1, 6).astype(np.int32)
        return dict(blocks=b, bpdx=1, bpdy=1, h0=1 / 8, level_max=6, rtol=0.7, ctol=0.35, linf=group_tags(b, 13),
                    fields=seeded_fields(len(b), 3))
    if name == "generated":           # a generated mesh with level jumps at the walls
        import amr_meshes as M
        bx, by, b, lmax = M.GENERATED["2x1_walls"]
        b = M.reference_order(b, bx, by, lmax + 1).astype(np.int32)
        return dict(blocks=b, bpdx=bx, bpdy=by, h0=1 / 8, level_max=lmax + 1, rtol=0.8, ctol=0.3, linf=group_tags(b, 5),
                    fields=seeded_fields(len(b), 4))
    if name == "flux":                # base-5 level on a 3x1 domain (1024 blocks per rank), a few refinements
        import amr_meshes as M
        b = M.reference_order(M.uniform_mesh(3, 1, 5), 3, 1, 7).astype(np.int32)
        linf = np.zeros(len(b))
        # three blocks refine on rank 0, two on rank 2 (none adjacent): 1033 / 1024 / 1030 new blocks, within 1 %, so the
        # flux branch moves (1033-1024)/4 = 2 blocks right from rank 0 and -(1024-1030)/4 = 1 block left from rank 2
        for k in (100, 400, 700, 2200, 2700):
            linf[k] = 1.0
        return dict(blocks=b, bpdx=3, bpdy=1, h0=1 / 8, level_max=7, rtol=0.5, ctol=-1.0, linf=linf,
                    fields=seeded_fields(len(b), 9))
    raise KeyError(name)


CASES = ("runsh", "runsh_device_tags", "three_level", "generated", "flux")


def split_group(blocks, new, base_left):
    """rank_begin [0, cut, nb] through a compressed group of blocks -> new: its base sibling left (or right) of the cut"""
    _, _, groups = classify(blocks, new)
    for g in groups.values():
        base, others = g[0], g[1:]
        if base_left and max(others) > base:
            return np.array([0, base + 1, len(blocks)], dtype=np.int64)
        if not base_left and min(others) < base:
            return np.array([0, base, len(blocks)], dtype=np.int64)
    return None


def empty_producer(blocks, new):
    """rank_begin [0, k, k+1, nb]: the middle rank holds one non-base sibling k of a compressed group, so it produces no new
    block (min n == 0)"""
    _, _, groups = classify(blocks, new)
    for g in groups.values():
        for k in g[1:]:
            if 0 < k < len(blocks) - 1:
                return np.array([0, k, k + 1, len(blocks)], dtype=np.int64)
    return None


def partitions(c, new):
    """{label: old rank_begin}: even and uneven cuts on 1..5 ranks, cuts through compressed groups, a producer-less rank"""
    nb = len(c["blocks"])
    out = {"1": np.array([0, nb], dtype=np.int64)}
    for W in (2, 3, 5):
        out[f"{W}even"] = np.array([nb * r // W for r in range(W + 1)], dtype=np.int64)
    out["4uneven"] = np.array([0, nb // 10, nb // 3, nb // 2 + 7, nb], dtype=np.int64)
    for label, rb in (("base_left", split_group(c["blocks"], new, True)), ("base_right", split_group(c["blocks"], new, False)),
                      ("empty", empty_producer(c["blocks"], new))):
        if rb is not None:
            out[label] = rb
    if len(c["blocks"]) == 3 * 1024:
        out = {"3flux": np.array([0, 1024, 2048, 3072], dtype=np.int64)}
    return out


# ---- one context's run -------------------------------------------------------------------------------------------------------
def run(sim, c, b0, b1, regrid_to=None, dist=None, steps=2):
    """upload the case's fields (blocks b0 .. b1), adapt (or regrid onto `regrid_to`), download, step: dict of results"""
    for n, a in c["fields"].items():
        sim.upload(n, a[b0:b1])
    linf = None if c["linf"] is None else c["linf"][b0:b1]
    if regrid_to is None:
        changed = sim.adapt(c["rtol"], c["ctol"], c["level_max"], block_linf=linf, dist=dist)
    else:
        sim.regrid(regrid_to, dist=dist)
        changed = None
    res = dict(changed=changed, blocks=sim.block_list(), rb=sim.rank_begin(), mine=sim.blocks.copy())
    res.update({n: sim.download(n) for n in FIELDS})
    res["steps"] = []
    for _ in range(steps):
        res["steps"].append(sim.step(cfl=0.5, max_iter=3))
        res["steps"][-1] = res["steps"][-1] + tuple(sim.download(n) for n in ("vel", "pres", "tmp"))
    return res


def one_rank(c, regrid_to=None, steps=2):
    from cup2d_b200.amr import AmrSimulation
    sim = AmrSimulation(c["blocks"], c["bpdx"], c["bpdy"], c["h0"], NU)
    sim.set_fast(True)
    r = run(sim, c, 0, len(c["blocks"]), regrid_to, steps=steps)
    sim.close()
    return r


def on_rank(c, rank, rb, dist, device=0, barrier=None, regrid_to=None, steps=2):
    from cup2d_b200.amr import AmrSimulation
    sim = AmrSimulation.distributed(c["blocks"], c["bpdx"], c["bpdy"], c["h0"], NU, rank, rb, dist, device=device)
    r = run(sim, c, int(rb[rank]), int(rb[rank + 1]), regrid_to, dist=dist, steps=steps)
    if barrier is not None:
        barrier()          # no rank frees its arrays while a peer may still read them
    sim.close()
    return r


def compare(c, one, parts, orb):
    """the ranks' results against the plain context's; returns the largest relative step difference"""
    W = len(parts)
    new = one["blocks"]
    want_rb = rule(produced(c["blocks"], new, orb))
    for p in parts:
        assert np.array_equal(p["blocks"], new)
        assert np.array_equal(p["rb"], want_rb), (p["rb"], want_rb)
        assert p["changed"] in (None, True) or W == 1 and not one["changed"]
    for n in MOVED:
        got = np.concatenate([p[n] for p in parts])
        assert np.array_equal(got, one[n]), n
    for p in parts:
        assert not p["tmpV"].any()
    worst = 0.0
    for k, s1 in enumerate(one["steps"]):
        for p in parts:
            assert p["steps"][k][0] == s1[0] if W == 1 else abs(p["steps"][k][0] - s1[0]) <= STEP_TOL * s1[0], (k, "dt")
        for q, name in enumerate(("vel", "pres", "tmp")):
            got, want = np.concatenate([p["steps"][k][3 + q] for p in parts]), s1[3 + q]
            d = float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-300))
            if W == 1:
                assert np.array_equal(got, want), (k, name)
            worst = max(worst, d)
    assert worst <= STEP_TOL, worst
    return worst


# ---- several GPUs: one process per rank under torch.distributed.run ----------------------------------------------------------
def main():
    import torch
    import torch.distributed as td
    td.init_process_group("gloo")
    rank, W = td.get_rank(), td.get_world_size()
    torch.cuda.set_device(rank)
    worst = 0.0
    for name in ("runsh", "runsh_device_tags", "three_level", "generated"):
        c = case(name)
        one = one_rank(c) if rank == 0 else None
        box = [one]
        td.broadcast_object_list(box, src=0)
        one = box[0]
        rb = np.array([len(c["blocks"]) * r // W for r in range(W + 1)], dtype=np.int64)
        r = on_rank(c, rank, rb, td, device=rank, barrier=td.barrier)
        parts = [None] * W
        td.all_gather_object(parts, r)
        if rank == 0:
            worst = max(worst, compare(c, one, parts, rb))
            print(f"{name}: {W} ranks {rb.tolist()} -> {parts[0]['rb'].tolist()} worst {worst:.3e}", flush=True)
    if rank == 0:
        print("ADAPT_RANKS_OK", worst, flush=True)
    td.destroy_process_group()


if __name__ == "__main__":
    main()
