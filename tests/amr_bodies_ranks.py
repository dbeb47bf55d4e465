"""The four body calls (cup2d_amr_ongrid, _surface, _forces, _collide) on distributed multi-level contexts
(cup2d_amr_create_ranks) against a one-rank cup2d_amr_create context on the same inputs.  Shared by
tests/test_amr_bodies_ranks_emulation.py (ranks as threads of one process, on the emulated library) and
tests/test_gpu_amr_bodies_ranks.py (one H100: a one-rank distributed context; several GPUs: run as a script under
torch.distributed.run, one process per GPU).

What is compared (a rank's results are its own blocks; shape and surface block ids are local and mapped to global here):
  bitwise, per rank           tmp, chi, every shape's ids, dist, chi and uncorrected u_def, the surface points, normals and
                              per-point skin values (but for the u_def columns after ongrid: those are the corrected u_def)
  to 1e-12 of the largest |value| of each quantity     Mass / COM, the seven sums, the corrected u_def, the 19 force sums and
                              the derived four, the collision sums and (u, v, omega) after the model
  bitwise across ranks        every scalar output; the impulse fires for the same pairs as on one rank
A one-rank distributed context is bitwise the plain context everywhere (its all-reduce is a no-op)."""
import os
import sys
import threading

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tools"), os.path.join(HERE, "golden")):
    if p not in sys.path:
        sys.path.insert(0, p)

import amr_body_oracle as bo  # noqa: E402

NU = 4e-5
RIGID = ("u", "v", "omega", "center_of_mass", "M", "J", "length")


# ---- inputs ------------------------------------------------------------------------------------------------------------
def _bodies(call):
    return [{**{n: s[n] for n in bo.MIDLINE}, "center": s["center"], "orientation": s["orientation"],
             "center_of_mass": s["center_of_mass"]} for s in call["shapes"]]


def seeded_fields(blocks, h0):
    """smooth vel [nb,8,8,2] and pres [nb,8,8,1] on the cell centres"""
    b = np.asarray(blocks)
    h = (h0 / (1 << b[:, 0]).astype(np.float64))[:, None, None]
    c = np.arange(8) + 0.5
    x = (b[:, 1, None, None] * 8 + c[None, None, :]) * h
    y = (b[:, 2, None, None] * 8 + c[None, :, None]) * h
    vel = np.stack([0.3 * np.sin(2.1 * x + 0.3) * np.cos(1.7 * y) + 0.05, 0.2 * np.cos(1.3 * x) * np.sin(2.3 * y + 0.1)], -1)
    return vel, (0.5 * np.cos(1.9 * x - 0.2) * np.cos(1.1 * y + 0.4))[..., None]


def case_inputs(name):
    """the inputs of one case: dict(kind, blocks, bpdx, bpdy, h0, nu, ...) (see chain())"""
    if name in ("runsh_ongrid", "synth_ongrid"):
        if name == "runsh_ongrid":
            import make_ongrid_golden
            c = make_ongrid_golden.load(os.path.join(HERE, "golden", "amrongrid_lmax8.npz"))[0]
            blocks, bpdx, bpdy, h0, bodies = c["blocks"], c["bpdx"], c["bpdy"], c["h0"], _bodies(c)
            want = dict(tmp=c["tmp"], chi=c["chi"], shapes=c["shapes"])
        else:   # three levels, two overlapping fish and one across the level interfaces
            import bench_amr
            blocks, bpdx, bpdy, h0 = bench_amr.three_level_mesh(3, r1=0.3, r2=0.15, centre=(0.45, 0.55)), 1, 1, 1 / 8
            bodies = [bo.synthetic_body((0.45, 0.55), 0.12, 97, 0.3, com_offset=(0.002, -0.001)),
                      bo.synthetic_body((0.47, 0.56), 0.10, 81, 2.5, bend=0.5, phase=1.0),
                      bo.synthetic_body((0.62, 0.55), 0.2, 161, -0.2)]
            want = bo.ongrid(blocks, bpdx, bpdy, h0, bodies)
        vel, pres = seeded_fields(blocks, h0)
        return dict(kind="ongrid", blocks=np.asarray(blocks, dtype=np.int32), bpdx=bpdx, bpdy=bpdy, h0=h0, nu=NU, bodies=bodies,
                    vel=vel, pres=pres, want=want)
    if name == "runsh_forces":
        import make_forces_golden
        st = make_forces_golden.load(os.path.join(HERE, "golden", "amrforces_lmax8.npz"))[0]
        return dict(kind="forces", blocks=st["blocks"], bpdx=st["bpdx"], bpdy=st["bpdy"], h0=st["h0"], nu=st["nu"],
                    chi=st["chi_n"], tmp=st["tmp"], vel=st["vel"], pres=st["pres"], shapes=st["shapes"], st=st)
    if name.startswith("runsh_collide"):
        import make_collide_golden
        c = make_collide_golden.load(os.path.join(HERE, "golden", "amrcollide_lmax8.npz"))[int(name[-1])]
        return dict(kind="collide", blocks=c["blocks"], bpdx=c["bpdx"], bpdy=c["bpdy"], h0=c["h0"], nu=NU, shapes=c["shapes"],
                    sums20=c["sums20"], uvw_after=c["uvw_after"])
    raise KeyError(name)


CASES = ("runsh_ongrid", "synth_ongrid", "runsh_forces", "runsh_collide0", "runsh_collide1", "runsh_collide2", "runsh_collide3")


# ---- one context's run -------------------------------------------------------------------------------------------------
def _motions_from(out10, length=0.2):
    return [{"u": o[7], "v": o[8], "omega": o[9], "center_of_mass": o[3:5], "M": o[5], "J": o[6], "length": length} for o in out10]


def chain(sim, inp, b0, b1):
    """the case's calls on `sim`, which holds blocks b0 .. b1 (the whole list on one rank); block ids in the results global"""
    sl, n8 = slice(b0, b1), None
    res = {}
    if inp["kind"] == "ongrid":
        sim.upload("vel", inp["vel"][sl])
        sim.upload("pres", inp["pres"][sl])
        out10 = sim.ongrid(inp["bodies"])
        n8 = len(inp["bodies"])
        sim.surface(n8)
        mo = _motions_from(out10)
        res.update(out10=out10, f23=sim.forces(mo))
        res["uvw"], res["sums20"] = sim.collide(mo)
        res["motions"] = np.array([[m["u"], m["v"], m["omega"]] for m in mo])
    elif inp["kind"] == "forces":
        sim.upload("chi", inp["chi"][sl])
        sim.upload("tmp", inp["tmp"][sl])
        for k, s in enumerate(inp["shapes"]):
            mine = (s["ids"] >= b0) & (s["ids"] < b1)
            sim.shape_set(k, s["ids"][mine] - b0, s["chi"][mine], s["udef"][mine])
        n8 = len(inp["shapes"])
        sim.surface(n8)
        sim.upload("vel", inp["vel"][sl])
        sim.upload("pres", inp["pres"][sl])
        res["f23"] = sim.forces(inp["shapes"])
    else:
        for k, s in enumerate(inp["shapes"]):
            mine = (s["ids"] >= b0) & (s["ids"] < b1)
            sim.shape_set(k, s["ids"][mine] - b0, s["chi"][mine], s["udef"][mine])
            sim.shape_set_dist(k, s["dist"][mine])
        mo = [{n: s[n] for n in RIGID} for s in inp["shapes"]]
        res["uvw"], res["sums20"] = sim.collide(mo)
        res["motions"] = np.array([[m["u"], m["v"], m["omega"]] for m in mo])
    res["tmp"], res["chi"] = sim.download("tmp")[..., 0], sim.download("chi")[..., 0]
    if inp["kind"] == "ongrid":
        res["shapes"] = []
        for k in range(n8):
            g = sim.shape_get(k)
            g["ids"] = g["ids"] + b0
            res["shapes"].append(g)
    if n8:
        res["surface"] = []
        for k in range(n8):
            g = sim.surface_get(k)
            g["block"] = g["block"] + b0
            res["surface"].append(g)
    return res


def one_rank(inp):
    """the plain context (cup2d_amr_create)"""
    from cup2d_b200.amr import AmrSimulation
    sim = AmrSimulation(inp["blocks"], inp["bpdx"], inp["bpdy"], inp["h0"], inp["nu"])
    r = chain(sim, inp, 0, len(inp["blocks"]))
    sim.close()
    return r


def on_rank(inp, rank, rb, dist, device=0, barrier=None):
    """this rank's share of a distributed context (cup2d_amr_create_ranks) and the case's calls on it"""
    from cup2d_b200.amr import AmrSimulation
    sim = AmrSimulation.distributed(inp["blocks"], inp["bpdx"], inp["bpdy"], inp["h0"], inp["nu"], rank, rb, dist, device=device)
    r = chain(sim, inp, int(rb[rank]), int(rb[rank + 1]))
    if barrier is not None:
        barrier()          # no rank frees its arrays while a peer may still read them
    sim.close()
    return r


class ThreadDist:
    """in-process stand-in for torch.distributed (carries the opaque peer blobs) for ranks running as threads"""
    def __init__(self, bar, slots, rank):
        self.bar, self.slots, self.rank = bar, slots, rank

    def all_gather_object(self, out, obj):
        self.slots[self.rank] = obj
        self.bar.wait()
        out[:] = self.slots
        self.bar.wait()

    def barrier(self):
        self.bar.wait()


def on_threads(W, fn):
    """fn(rank, dist, barrier) on W threads; returns the W results (raises the first error)"""
    bar, slots, res, errs = threading.Barrier(W), [None] * W, [None] * W, []

    def run(rank):
        try:
            res[rank] = fn(rank, ThreadDist(bar, slots, rank), bar.wait)
        except Exception as e:  # noqa: BLE001 - reported below
            errs.append(f"rank {rank}: {e!r}")
            bar.abort()
    ths = [threading.Thread(target=run, args=(r,)) for r in range(W)]
    [t.start() for t in ths]
    [t.join() for t in ths]
    if errs:
        raise RuntimeError("; ".join(errs))
    return res


# ---- partitions ----------------------------------------------------------------------------------------------------------
def obstacle_ids(inp, one):
    if inp["kind"] == "ongrid":
        return [np.asarray(s["ids"]) for s in one["shapes"]]
    return [np.asarray(s["ids"]) for s in inp["shapes"]]


def partitions(inp, one):
    """{W: rank_begin} for 1..4 ranks: 2 cuts through the first shape's obstacle blocks (or, for a colliding pair, through
    their common blocks); 3 gives one rank no obstacle block and another the whole first shape; 4 cuts the obstacle blocks
    of all shapes at their quartiles"""
    nb = len(inp["blocks"])
    ids = obstacle_ids(inp, one)
    allids = np.unique(np.concatenate(ids))
    first = np.sort(ids[0])
    if inp["kind"] == "collide":
        common = np.intersect1d(ids[0], ids[1])
        if len(common) >= 2:
            first = common
    out = {1: [0, nb], 2: [0, int(first[len(first) // 2]), nb]}
    lo, hi0 = int(allids[0]), int(first[-1]) + 1
    if lo > 0 and hi0 < nb:                       # rank 0: the blocks before every obstacle block
        out[3] = [0, lo, hi0, nb]
    else:                                         # the widest gap between obstacle blocks
        gaps = np.diff(np.concatenate([[-1], allids, [nb]]))
        g = int(np.argmax(gaps))
        a, b = int(np.concatenate([[-1], allids])[g]) + 1, int(np.concatenate([allids, [nb]])[g])
        out[3] = sorted({0, a, b, nb}) if a > 0 and b < nb else [0, a, b, nb] if a > 0 else [0, b, (b + nb) // 2, nb]
    q = [int(allids[len(allids) * k // 4]) for k in (1, 2, 3)]
    out[4] = [0] + q + [nb]
    for W, rb in out.items():
        assert len(rb) == W + 1 and all(rb[r] < rb[r + 1] for r in range(W)), (W, rb)
    return {W: np.array(rb, dtype=np.int64) for W, rb in out.items()}


def properties(inp, one, parts):
    """which of the partitions' required properties hold: a rank with no obstacle block, a shape entirely on one rank, an
    irregular obstacle block whose kind-2 (chi) or kind-3 (force) lab reads a block of another rank, a colliding pair's
    common blocks on several ranks"""
    from cup2d_b200.amr import AmrPlan
    ids = obstacle_ids(inp, one)
    allids = np.unique(np.concatenate(ids))
    plan = AmrPlan(inp["blocks"], inp["bpdx"], inp["bpdy"])
    irr = plan.irregular()
    remote_srcs = {}
    for which, ncell in ((2, 100), (3, 256)):
        rp, dst, sb, _, _ = plan.ghosts(which)
        blk = irr[dst // ncell]
        rows_of = np.repeat(blk, np.diff(rp))
        remote_srcs[which] = (rows_of, sb)
    plan.close()
    prop = dict(empty_rank=False, whole_shape=False, remote_level_jump=False, split_common=False)
    for W, rb in parts.items():
        owner = np.searchsorted(rb, np.arange(len(inp["blocks"])), side="right") - 1
        if W > 1:
            prop["empty_rank"] |= any(not ((allids >= rb[r]) & (allids < rb[r + 1])).any() for r in range(W))
            prop["whole_shape"] |= any(len(np.unique(owner[s])) == 1 for s in ids if len(s))
            for rows_of, sb in remote_srcs.values():
                on_ob = np.isin(rows_of, allids)
                prop["remote_level_jump"] |= bool((owner[rows_of[on_ob]] != owner[sb[on_ob]]).any())
            if len(ids) > 1:
                common = np.intersect1d(ids[0], ids[1])
                prop["split_common"] |= len(np.unique(owner[common])) > 1
    return prop


# ---- comparison ----------------------------------------------------------------------------------------------------------
def _rel(got, want):
    """max |got - want| over each quantity's largest |want| (columns of the last axis)"""
    got, want = np.atleast_2d(got), np.atleast_2d(want)
    scale = np.abs(want).max(axis=0)
    d = np.abs(got - want).max(axis=0)
    return float(np.max(np.where(scale > 0, d / np.where(scale > 0, scale, 1), d)))


def compare(one, parts, rb, tol=1e-12):
    """the distributed results `parts` (one per rank) against the plain context's `one`; returns the largest relative
    difference of the quantities that agree to rounding"""
    W = len(parts)
    worst = 0.0
    for name in ("tmp", "chi"):
        assert np.array_equal(np.concatenate([p[name] for p in parts]), one[name]), name
    for k, s1 in enumerate(one.get("shapes", [])):
        got = {n: np.concatenate([p["shapes"][k][n] for p in parts]) for n in ("ids", "dist", "chi", "udef")}
        for n in ("ids", "dist", "chi"):
            assert np.array_equal(got[n], s1[n]), (k, n)
        worst = max(worst, float(np.abs(got["udef"] - s1["udef"]).max(initial=0.0) / max(np.abs(s1["udef"]).max(initial=0.0), 1e-300)))
    for k, s1 in enumerate(one.get("surface", [])):
        for n in ("block", "ixy", "normal"):
            assert np.array_equal(np.concatenate([p["surface"][k][n] for p in parts]), s1[n]), (k, n)
        skin = np.concatenate([p["surface"][k]["skin"] for p in parts])
        # after ongrid the skin's u_def columns (uDef_s, vDef_s) are the corrected u_def: to rounding
        udef_cols = [8, 9] if "shapes" in one else []
        keep = [c for c in range(14) if c not in udef_cols]
        assert np.array_equal(skin[:, keep], s1["skin"][:, keep]), k
        if udef_cols:
            worst = max(worst, _rel(skin[:, udef_cols], s1["skin"][:, udef_cols]))
    for name in ("out10", "f23", "sums20", "uvw"):
        if name not in one:
            continue
        for p in parts[1:]:
            assert np.array_equal(p[name], parts[0][name]), f"{name} differs across ranks"
        worst = max(worst, _rel(parts[0][name], one[name]))
    if W == 1:           # one rank: the all-reduce is a no-op, every result is the plain context's bit for bit
        for name in ("out10", "f23", "sums20", "uvw"):
            assert name not in one or np.array_equal(parts[0][name], one[name]), name
        for k, s1 in enumerate(one.get("shapes", [])):
            assert np.array_equal(parts[0]["shapes"][k]["udef"], s1["udef"]), k
        for k, s1 in enumerate(one.get("surface", [])):
            assert np.array_equal(parts[0]["surface"][k]["skin"], s1["skin"]), k
    if "uvw" in one:     # the impulse fires for the same pairs
        assert np.array_equal(parts[0]["uvw"] != parts[0]["motions"], one["uvw"] != one["motions"])
    assert worst <= tol, worst
    return worst


def assemble(parts):
    """the ranks' results as one: fields, shapes and surface points concatenated in rank order, scalars of rank 0"""
    out = dict(parts[0])
    for name in ("tmp", "chi"):
        out[name] = np.concatenate([p[name] for p in parts])
    for key in ("shapes", "surface"):
        if key in out:
            out[key] = [{n: np.concatenate([p[key][k][n] for p in parts]) for n in parts[0][key][k] if parts[0][key][k][n] is not None}
                        for k in range(len(out[key]))]
    return out


def udef_pre_replay(res, want_shapes, blocks, h0):
    """u_def before the correction, bitwise: the call's own correction replayed in numpy on the pinned uncorrected u_def"""
    for k, w in enumerate(want_shapes):
        g, o = res["shapes"][k], res["out10"][k]
        b = np.asarray(blocks)[w["ids"]]
        h = (h0 / (1 << b[:, 0]).astype(np.float64))[:, None, None]
        c = np.arange(8) + 0.5
        x = (b[:, 1, None, None] * 8).astype(np.float64) * h + h * c[None, None, :] + 0 * c[None, :, None]
        y = (b[:, 2, None, None] * 8).astype(np.float64) * h + h * c[None, :, None] + 0 * c[None, None, :]
        px, py = x - o[3], y - o[4]
        pre = w["udef_pre"]
        replay = np.stack([pre[..., 0] - (o[7] - o[9] * py), pre[..., 1] - (o[8] + o[9] * px)], axis=-1)
        assert np.array_equal(g["ids"], w["ids"]) and np.array_equal(g["udef"], replay), k


def check_pinned(inp, res):
    """the distributed results against the numbers the existing oracles pin (tests/golden, tests/amr_*_oracle.py), with
    the tolerances of the one-rank tests"""
    if inp["kind"] == "ongrid":
        want = inp["want"]
        assert np.array_equal(res["tmp"], want["tmp"])
        assert np.abs(res["chi"] - want["chi"]).max() <= 1e-13
        for k, w in enumerate(want["shapes"]):
            assert np.array_equal(res["shapes"][k]["dist"], w["dist"])
            o, q = res["out10"][k], w["sums7"]
            assert np.all(np.abs(o[:3] - w["com3"]) <= 1e-12 * np.abs(w["com3"]))
            assert abs(o[5] - q[2]) <= 1e-12 * abs(q[2]) and abs(o[6] - q[3]) <= 1e-12 * abs(q[3])
        udef_pre_replay(res, want["shapes"], inp["blocks"], inp["h0"])
    elif inp["kind"] == "forces":
        for k, s in enumerate(inp["shapes"]):
            scale = np.maximum(np.abs(s["q19"]), np.abs(s["acc"]).sum(axis=0))
            assert (np.abs(res["f23"][k, :19] - s["q19"]) <= 1e-12 * scale).all(), k
    else:
        scale = np.maximum(np.abs(inp["sums20"]).max(axis=0), 1e-300)
        assert (np.abs(res["sums20"] - inp["sums20"]) <= 1e-12 * scale).all()
        assert np.array_equal(res["uvw"] != res["motions"], inp["uvw_after"] != res["motions"])
        assert np.abs(res["uvw"] - inp["uvw_after"]).max() <= 1e-12 * max(np.abs(inp["uvw_after"]).max(), 1e-300)


# ---- several GPUs: one process per rank under torch.distributed.run ----------------------------------------------------
def main():
    import torch
    import torch.distributed as td
    td.init_process_group("gloo")
    rank, W = td.get_rank(), td.get_world_size()
    torch.cuda.set_device(rank)
    worst = 0.0
    for name in ("runsh_ongrid", "synth_ongrid", "runsh_forces", "runsh_collide0"):
        inp = case_inputs(name)
        one = one_rank(inp) if rank == 0 else None
        one = [one]
        td.broadcast_object_list(one, src=0)
        one = one[0]
        rb = partitions(inp, one)[min(W, 4)] if W <= 4 else np.array([len(inp["blocks"]) * r // W for r in range(W + 1)])
        r = on_rank(inp, rank, rb, td, device=rank, barrier=td.barrier)
        parts = [None] * W
        td.all_gather_object(parts, r)
        if rank == 0:
            worst = max(worst, compare(one, parts, rb))
            print(f"{name}: {W} ranks {rb.tolist()} worst {worst:.3e}", flush=True)
    if rank == 0:
        print("BODIES_RANKS_OK", worst, flush=True)
    td.destroy_process_group()


if __name__ == "__main__":
    main()
