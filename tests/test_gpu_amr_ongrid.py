"""GPU tests of ongrid() on multi-level contexts (cup2d_amr_ongrid, csrc/amr_ongrid.cu): against the reference's own ongrid()
on its run.sh mesh (tests/golden/amrongrid_lmax8.npz) and against the oracle (tests/amr_body_oracle.py) on synthetic
three-level meshes.  They also pass on the CPU against the emulated build of the same sources (tests/test_amr_ongrid.py)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import amr_body_oracle as bo

pytestmark = [pytest.mark.gpu]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def calls(golden_dir):
    sys.path.insert(0, golden_dir)
    import make_ongrid_golden
    return make_ongrid_golden.load(os.path.join(golden_dir, "amrongrid_lmax8.npz"))


def _bodies(call):
    return [{**{n: s[n] for n in bo.MIDLINE}, "center": s["center"], "orientation": s["orientation"],
             "center_of_mass": s["center_of_mass"]} for s in call["shapes"]]


def _sim(blocks, bpdx, bpdy, h0):
    from cup2d_b200.amr import AmrSimulation
    return AmrSimulation(blocks, bpdx, bpdy, h0, 4e-5)


def _copy_only(blocks, bpdx, bpdy):
    """blocks whose +-1 scalar lab (kind 2) is plain copies: their chi is bitwise the reference's"""
    from cup2d_b200.amr import AmrPlan
    p = AmrPlan(blocks, bpdx, bpdy)
    rowptr, _, _, w = p.stencil(2)
    p.close()
    n = np.diff(rowptr).reshape(len(blocks), 10, 10)
    first = w[np.minimum(rowptr[:-1], len(w) - 1)].reshape(len(blocks), 10, 10)
    ok = ((n == 1) & (first == 1.0)) | (n == 0)
    return ok.reshape(len(blocks), -1).all(axis=1)


def _block_xy(blocks, h0, ids):
    b = np.asarray(blocks)[ids]
    h = h0 / (1 << b[:, 0]).astype(np.float64)
    c = np.arange(8) + 0.5
    x = (b[:, 1] * 8).astype(np.float64)[:, None, None] * h[:, None, None] + h[:, None, None] * c[None, None, :] + 0 * c[None, :, None]
    y = (b[:, 2] * 8).astype(np.float64)[:, None, None] * h[:, None, None] + h[:, None, None] * c[None, :, None] + 0 * c[None, None, :]
    return x, y


def _check(sim, out, want, blocks, bpdx, bpdy, h0):
    """sim after ongrid against `want` (the fixture's call or the oracle's result), with the tolerances of the header"""
    exact = _copy_only(blocks, bpdx, bpdy)
    assert np.array_equal(sim.download("tmp")[..., 0], want["tmp"])
    chi = sim.download("chi")[..., 0]
    assert np.array_equal(chi[exact], want["chi"][exact])
    assert np.abs(chi - want["chi"]).max() <= 1e-13
    for k, w in enumerate(want["shapes"]):
        g = sim.shape_get(k)
        assert np.array_equal(g["ids"], w["ids"])
        assert np.array_equal(g["dist"], w["dist"])
        ex = exact[w["ids"]]
        assert np.array_equal(g["chi"][ex], w["chi"][ex]) and np.abs(g["chi"] - w["chi"]).max() <= 1e-13
        com3, q = w["com3"], w["sums7"]
        assert np.all(np.abs(out[k, :3] - com3) <= 1e-12 * np.abs(com3)), (out[k, :3], com3)
        assert np.all(np.abs(out[k, 3:5] - w["new_center_of_mass"]) <= 1e-14 * np.abs(w["new_center_of_mass"]))
        m, j, u, v, a = q[2], q[3], q[4] / q[2], q[5] / q[2], q[6] / q[3]
        assert abs(out[k, 5] - m) <= 1e-12 * abs(m) and abs(out[k, 6] - j) <= 1e-12 * abs(j)
        for got, ref, scale in ((out[k, 7], u, abs(q[4]) / m), (out[k, 8], v, abs(q[5]) / m), (out[k, 9], a, abs(q[6]) / j)):
            assert abs(got - ref) <= 1e-12 * max(scale, 1e-300)
        # u_def before the correction, bitwise: the device's correction replayed in numpy on the reference's u_def
        x, y = _block_xy(blocks, h0, w["ids"])
        cmx, cmy = out[k, 3], out[k, 4]
        px, py = x - cmx, y - cmy
        pre = w["udef_pre"]
        replay = np.stack([pre[..., 0] - (out[k, 7] - out[k, 9] * py), pre[..., 1] - (out[k, 8] + out[k, 9] * px)], axis=-1)
        assert np.array_equal(g["udef"], replay)
        assert np.abs(g["udef"] - w["udef"]).max() <= 1e-13 * np.abs(w["udef"]).max()


def test_ongrid_reproduces_the_reference(calls):
    for c in calls:
        sim = _sim(c["blocks"], c["bpdx"], c["bpdy"], c["h0"])
        out = sim.ongrid(_bodies(c))
        want = dict(tmp=c["tmp"], chi=c["chi"], shapes=c["shapes"])
        for s in c["shapes"]:
            assert len(s["ids"]) > 20
        _check(sim, out, want, c["blocks"], c["bpdx"], c["bpdy"], c["h0"])
        sim.close()


def test_two_calls_are_bitwise_identical(calls):
    c = calls[0]
    sim = _sim(c["blocks"], c["bpdx"], c["bpdy"], c["h0"])
    sim.upload("chi", np.random.default_rng(0).uniform(0, 1, (len(c["blocks"]), 8, 8, 1)))   # overwritten by the call
    o1 = sim.ongrid(_bodies(c))
    r1 = [sim.download("chi"), sim.download("tmp")] + [sim.shape_get(k) for k in range(2)]
    o2 = sim.ongrid(_bodies(c))
    r2 = [sim.download("chi"), sim.download("tmp")] + [sim.shape_get(k) for k in range(2)]
    assert np.array_equal(o1, o2)
    assert np.array_equal(r1[0], r2[0]) and np.array_equal(r1[1], r2[1])
    for a, b in zip(r1[2:], r2[2:]):
        for n in a:
            assert np.array_equal(a[n], b[n]), n
    sim.close()


def test_downstream_calls_equal_shape_set(calls):
    """shape_integrals / penalize / udef_assemble after ongrid equal the same calls after shape_set of the blocks ongrid left
    on the device (read back with shape_get): the storage ongrid writes is the storage the downstream calls read.  That those
    blocks are the reference's is test_ongrid_reproduces_the_reference."""
    c = calls[0]
    nb = len(c["blocks"])
    rng = np.random.default_rng(3)
    vel = rng.uniform(-1, 1, (nb, 8, 8, 2))
    a = _sim(c["blocks"], c["bpdx"], c["bpdy"], c["h0"])
    a.upload("vel", vel)
    out = a.ongrid(_bodies(c))
    b = _sim(c["blocks"], c["bpdx"], c["bpdy"], c["h0"])
    b.upload("vel", vel)
    b.upload("chi", a.download("chi"))
    for k in range(2):
        g = a.shape_get(k)
        b.shape_set(k, g["ids"], g["chi"], g["udef"])
        with pytest.raises(Exception):
            b.shape_get(k)        # a shape set from the host has no dist
        assert np.array_equal(b.shape_get(k, dist=False)["udef"], g["udef"])
    for k in range(2):
        args = (k, 1e7, 1e-4, out[k, 3], out[k, 4])
        assert np.array_equal(a.shape_integrals(*args), b.shape_integrals(*args))
        a.penalize(*args, 0.1, -0.05, 0.3)
        b.penalize(*args, 0.1, -0.05, 0.3)
    a.udef_assemble()
    b.udef_assemble()
    assert np.array_equal(a.download("vel"), b.download("vel"))
    assert np.array_equal(a.download("tmpV"), b.download("tmpV"))
    assert np.abs(a.download("tmpV")).max() > 0
    a.close()
    b.close()


def test_regrid_clears_shapes_and_ongrid_matches_a_fresh_context(calls):
    from cup2d_b200.amr import adapt_mesh
    c = calls[0]
    blocks = c["blocks"]
    sim = _sim(blocks, c["bpdx"], c["bpdy"], c["h0"])
    sim.ongrid(_bodies(c))
    linf = np.zeros(len(blocks))
    linf[np.flatnonzero(blocks[:, 0] == 6)[:8]] = 1.0     # level 7 (levelMax - 1) is the finest
    new = adapt_mesh(blocks, c["bpdx"], c["bpdy"], 8, linf, 0.5, 0.0)
    assert len(new) > len(blocks)
    sim.regrid(new)
    with pytest.raises(Exception):
        sim.shape_get(0)
    o1 = sim.ongrid(_bodies(c))
    fresh = _sim(new, c["bpdx"], c["bpdy"], c["h0"])
    o2 = fresh.ongrid(_bodies(c))
    assert np.array_equal(o1, o2)
    for n in ("chi", "tmp"):
        assert np.array_equal(sim.download(n), fresh.download(n))
    for k in range(2):
        g1, g2 = sim.shape_get(k), fresh.shape_get(k)
        for n in g1:
            assert np.array_equal(g1[n], g2[n])
    sim.close()
    fresh.close()


def test_error_paths_leave_the_context_unchanged(calls):
    from cup2d_b200 import lib as L
    c = calls[0]
    sim = _sim(c["blocks"], c["bpdx"], c["bpdy"], c["h0"])
    sim.ongrid(_bodies(c))
    before = [sim.download("chi"), sim.download("tmp"), sim.shape_get(0), sim.shape_get(1)]
    bad = _bodies(c)
    bad[1] = dict(bad[1], center=np.array([-0.1, 0.5]))
    with pytest.raises(L.Cup2dError, match="outside the domain"):
        sim.ongrid(bad)
    short = _bodies(c)
    short[0] = {n: (v[:5] if n in bo.MIDLINE else v) for n, v in short[0].items()}
    with pytest.raises(L.Cup2dError, match="nm >= 9"):
        sim.ongrid(short)
    after = [sim.download("chi"), sim.download("tmp"), sim.shape_get(0), sim.shape_get(1)]
    assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1])
    for a, b in zip(before[2:], after[2:]):
        for n in a:
            assert np.array_equal(a[n], b[n])
    rb = np.array([0, len(c["blocks"]) // 2, len(c["blocks"])], dtype=np.int64)
    L.check(sim.lib.cup2d_amr_set_ranks(sim._h, 0, 2, rb.ctypes.data_as(C.POINTER(C.c_int64))))
    out = np.empty(20)
    structs = (L.Body * 1)()
    assert sim.lib.cup2d_amr_ongrid(sim._h, 1, structs, out.ctypes.data_as(C.POINTER(C.c_double))) == -4
    sim.close()


def _three_level(base, centre=(0.45, 0.55)):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import bench_amr
    return bench_amr.three_level_mesh(base, r1=0.3, r2=0.15, centre=centre)


SYNTH = {
    # two overlapping fish in the finest region: tmp and chi take maxima across the shapes
    "overlapping": lambda: [bo.synthetic_body((0.45, 0.55), 0.12, 97, 0.3, com_offset=(0.002, -0.001)),
                            bo.synthetic_body((0.47, 0.56), 0.10, 81, 2.5, bend=0.5, phase=1.0)],
    # a fish across the level interfaces (finest -> middle -> base level)
    "level_jumps": lambda: [bo.synthetic_body((0.62, 0.55), 0.2, 161, -0.2)],
    # a vertical fish along the x = 0 wall: its smoothing band (|dist| <= h) reaches the wall column, whose chi reads the
    # wall ghosts of the tmp lab (main.cpp:3239-3244)
    # (on a mesh whose finest region touches that wall)
    "near_wall": lambda: [bo.synthetic_body((0.008, 0.6), 0.15, 121, 1.5708, bend=0.1)],
    # a long midline: Nsegments = 70 > 64
    "many_segments": lambda: [bo.synthetic_body((0.45, 0.5), 0.25, 8 * 70 + 1, 0.7, bend=0.8)],
}


@pytest.mark.parametrize("case", sorted(SYNTH))
def test_synthetic_three_level_ongrid_vs_oracle(case):
    base, h0 = 3, 1 / 8
    blocks = _three_level(base, (0.1, 0.6) if case == "near_wall" else (0.45, 0.55))
    bodies = SYNTH[case]()
    want = bo.ongrid(blocks, 1, 1, h0, bodies)
    levels = {int(blocks[k, 0]) for s in want["shapes"] for k in s["ids"]}
    if case == "level_jumps":
        assert len(levels) >= 2
    if case == "near_wall":   # cells of the smoothing band in column ix = 0 of blocks at the wall
        s = want["shapes"][0]
        h = h0 / (1 << blocks[s["ids"], 0]).astype(np.float64)
        band = np.abs(s["dist"][:, :, 0]) <= h[:, None]          # [nob, iy] at ix = 0
        at_wall = blocks[s["ids"], 1] == 0
        assert (band & at_wall[:, None]).sum() >= 4 and s["chi"][at_wall][:, :, 0].max() > 0
    if case == "overlapping":
        assert len(set(want["shapes"][0]["ids"].tolist()) & set(want["shapes"][1]["ids"].tolist())) > 4
    sim = _sim(blocks, 1, 1, h0)
    out = sim.ongrid(bodies)
    _check(sim, out, want, blocks, 1, 1, h0)
    sim.close()


def test_ongrid_timing(calls):
    """cup2d_amr_ongrid_timing / _times: CUDA-event times of the last call, every kernel class inside the whole call"""
    c = calls[0]
    sim = _sim(c["blocks"], c["bpdx"], c["bpdy"], c["h0"])
    from cup2d_b200 import lib as L
    with pytest.raises(L.Cup2dError):
        sim.ongrid_times()
    sim.ongrid_timing(True)
    o1 = sim.ongrid(_bodies(c))
    t = sim.ongrid_times()
    assert set(t) == set(sim.ONGRID_TIMES) and all(v >= 0 for v in t.values())
    assert sum(v for k, v in t.items() if k != "call") <= t["call"] + 1e-3
    sim.ongrid_timing(False)
    assert np.array_equal(sim.ongrid(_bodies(c)), o1)
    sim.close()
