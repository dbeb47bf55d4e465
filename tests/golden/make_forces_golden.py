"""Generate tests/golden/amrforces_lmax8.npz: the reference's own surface normals (ComputeSurfaceNormals, main.cpp:3774-3828)
and force diagnostics (KernelComputeForces, 5573-5746, and 7188-7284) on its run.sh case (tests/golden/ref_forces.cpp).

Run in the build container (needs /root/reference, which does not exist on the GPU box):

    python tests/golden/make_forces_golden.py

ref_forces.cpp includes the unmodified reference main.cpp and is compiled here with the reference's flags (those of
oracle/Makefile) into a temporary directory.  Two consecutive time steps of the run.sh case (levelMax 8, two fish, one OpenMP
thread).  Per step: the mesh, chi and tmp as the normals saw them, vel and pres as the forces saw them, at the first step
the reference's own VectorLab of vel and ScalarLab of chi (stencil {-4,-4,5,5,tensorial}) of every obstacle block with
surface points, and per shape the obstacle ids, chi and udef, u, v, centerOfMass, the surface points (ix, iy, dchidx,
dchidy, delta), the 14 skin arrays, the 19 per-block accumulators, the 19-value buffer and Pthrust, Pdrag, EffPDef,
EffPDefBnd.  load() gives a list of steps.

To keep the fixture small it holds only what the forces read: vel on the 3 x 3 block neighbourhoods (at any level) of the
obstacle blocks with surface points and pres on those blocks, zero elsewhere; and of the skin arrays the five that are
computed (omega_s, fX_s, fY_s, fXv_s, fYv_s).  The other nine are copies of recorded values (x_s, y_s the cell centre,
p_s = pres, u_s, v_s = vel, nx_s, ny_s the unit normal, uDef_s, vDef_s = udef at the point); the generator checks them
against the record bit for bit before dropping them, and load() rebuilds them with the reference's expressions.
"""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("CUP2D_REFERENCE", "/root/reference")
LEVEL_MAX, FIRST, COUNT = 8, 3, 2
OUT = os.path.join(HERE, f"amrforces_lmax{LEVEL_MAX}.npz")
SKIN_KEPT = (7, 10, 11, 12, 13)  # omega_s, fX_s, fY_s, fXv_s, fYv_s: the skin columns the fixture stores


def skin_copies(blocks, h0, vel, pres, s):
    """the nine skin columns that copy recorded values (main.cpp:5704-5713), by the reference's expressions: [n, 14] with the
    stored columns zero"""
    ids = np.repeat(np.asarray(s["ids"]), np.asarray(s["npts"]))
    q = np.repeat(np.arange(len(s["ids"])), np.asarray(s["npts"]))
    ix, iy = s["surf"][:, 0].astype(np.int64), s["surf"][:, 1].astype(np.int64)
    lvl, bi, bj = (blocks[ids, c].astype(np.int64) for c in range(3))
    h = h0 / (1 << lvl).astype(np.float64)                      # Info::h (main.cpp:693)
    o0 = (bi * 8) * h0 / (1 << lvl).astype(np.float64)          # Info::origin (695-696)
    o1 = (bj * 8) * h0 / (1 << lvl).astype(np.float64)
    nX, nY = s["surf"][:, 2], s["surf"][:, 3]
    norm = 1.0 / np.sqrt(nX * nX + nY * nY)
    out = np.zeros((len(ids), 14))
    out[:, 0], out[:, 1] = o0 + h * (ix + 0.5), o1 + h * (iy + 0.5)
    out[:, 2] = pres[ids, iy, ix]
    out[:, 3], out[:, 4] = vel[ids, iy, ix, 0], vel[ids, iy, ix, 1]
    out[:, 5], out[:, 6] = nX * norm, nY * norm
    out[:, 8], out[:, 9] = s["udef"][q, iy, ix, 0], s["udef"][q, iy, ix, 1]
    return out


def compile_harness(tmp):
    flags = ["-O3", "-fopenmp", "-std=c++17", "-D_BS_=8", "-include", "cfloat", "-I", os.path.join(ROOT, "oracle", "shim"),
             "-I", REF, "-w"]
    objs = []
    for src in (os.path.join(HERE, "ref_forces.cpp"), os.path.join(ROOT, "oracle", "ref_spmat_cpu.cpp")):
        o = os.path.join(tmp, os.path.basename(src) + ".o")
        subprocess.run(["/usr/bin/g++", *flags, "-c", src, "-o", o], check=True)
        objs.append(o)
    exe = os.path.join(tmp, "ref_forces")
    subprocess.run(["/usr/bin/g++", "-fopenmp", "-o", exe, *objs], check=True)
    return exe


def records(path):
    """the record stream split into steps: list of {tag: array}"""
    a = np.fromfile(path)
    i, steps = 0, []
    while i < len(a):
        tag, n = int(a[i]), int(a[i + 1])
        if tag == 1:
            steps.append({})
        steps[-1][tag] = a[i + 2:i + 2 + n]
        i += 2 + n
    return steps


def load(path=OUT):
    """list of steps; a step is a dict with blocks, bpdx, bpdy, h0, nu, chi_n / tmp (the normals' inputs), vel, pres, chi,
    lab_ids and (first step only) lab_vel [n, 16, 16, 2], lab_chi [n, 16, 16] and `shapes`, a list of per-shape dicts (ids, chi, udef, u, v,
    center_of_mass, npts [nob], surf [n, 5], skin [n, 14], acc [nob, 19], q19, derived4)"""
    d = dict(np.load(path))
    out = []
    for c in range(int(d["nsteps"])):
        p = f"c{c}_"
        st = {k[len(p):]: v for k, v in d.items() if k.startswith(p) and "_s" not in k[len(p):]}
        st.update(bpdx=int(d["bpdx"]), bpdy=int(d["bpdy"]), h0=float(d["h0"]), nu=float(d["nu"]))
        st["shapes"] = []
        for k in range(int(d["nshapes"])):
            q = f"{p}s{k}_"
            s = {key[len(q):]: v for key, v in d.items() if key.startswith(q)}
            s.update(center_of_mass=np.array([float(s.pop("cmx")), float(s.pop("cmy"))]), u=float(s["u"]), v=float(s["v"]))
            s["skin"] = skin_copies(st["blocks"], st["h0"], st["vel"], st["pres"], s)
            s["skin"][:, SKIN_KEPT] = s.pop("skin5")
            st["shapes"].append(s)
        out.append(st)
    return out


def main():
    if not os.path.exists(os.path.join(REF, "main.cpp")):
        sys.exit(f"the reference sources are needed: {REF}/main.cpp")
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        exe = compile_harness(tmp)
        fout = os.path.join(tmp, "forces.bin")
        subprocess.run([exe, str(LEVEL_MAX), str(FIRST), str(COUNT), fout], check=True, stdout=subprocess.DEVNULL,
                       stderr=subprocess.DEVNULL, env=dict(os.environ, OMP_NUM_THREADS="1"))
        steps = records(fout)
    assert len(steps) == COUNT, len(steps)
    jumps = []
    for c, r in enumerate(steps):
        step, ns, h0, bpdx, bpdy, nu = r[1]
        ns = int(ns)
        out.update(nshapes=ns, h0=h0, bpdx=int(bpdx), bpdy=int(bpdy), nu=nu)
        p = f"c{c}_"
        blocks = r[2].reshape(-1, 3).astype(np.int32)
        nb = len(blocks)
        out[p + "step"] = int(step)
        out[p + "blocks"] = blocks
        out[p + "chi_n"] = r[3].reshape(nb, 8, 8)
        out[p + "tmp"] = r[4].reshape(nb, 8, 8)
        chi = r[7].reshape(nb, 8, 8)
        assert np.array_equal(chi, out[p + "chi_n"]), "chi changed between the normals and the forces"
        lab_all = r[8].astype(np.int32)
        pointed = np.zeros(nb, dtype=bool)  # obstacle blocks with surface points: the only ones the forces read a lab of
        for k in range(ns):
            pointed[r[100 * k + 20].astype(np.int64)[r[100 * k + 21] > 0]] = True
        lab_ids = np.flatnonzero(pointed).astype(np.int32)
        # vel is kept on every block that meets the 3 x 3 block neighbourhood of one of them (at any level), pres on them
        near = np.zeros(nb, dtype=bool)
        lo, hi = blocks[:, 1:] * (1 << (16 - blocks[:, :1])), (blocks[:, 1:] + 1) * (1 << (16 - blocks[:, :1]))
        for k in lab_ids:
            w = 1 << (16 - int(blocks[k, 0]))
            near |= ((lo < hi[k] + w) & (hi > lo[k] - w)).all(axis=1)
        out[p + "vel"] = np.where(near[:, None, None, None], r[5].reshape(nb, 8, 8, 2), 0.0)
        out[p + "pres"] = np.where(pointed[:, None, None], r[6].reshape(nb, 8, 8), 0.0)
        out[p + "lab_ids"] = lab_ids
        if c == 0:  # the reference's own labs, of the first step
            sel = np.searchsorted(lab_all, lab_ids)
            assert np.array_equal(lab_all[sel], lab_ids)
            out[p + "lab_vel"] = r[9].reshape(len(lab_all), 16, 16, 2)[sel]
            out[p + "lab_chi"] = r[10].reshape(len(lab_all), 16, 16)[sel]
        # obstacle blocks whose 16 x 16 lab reaches a block of another level (any of the 8 neighbours is not same-level)
        index = {tuple(b): k for k, b in enumerate(blocks.tolist())}
        nx = lambda l: int(bpdx) << l
        ny = lambda l: int(bpdy) << l
        cross = 0
        for k in lab_ids:
            l, i, j = blocks[k]
            for di in (-1, 0, 1):
                for dj in (-1, 0, 1):
                    ii, jj = i + di, j + dj
                    if (di or dj) and 0 <= ii < nx(l) and 0 <= jj < ny(l) and (l, ii, jj) not in index:
                        cross += 1
                        break
                else:
                    continue
                break
        jumps.append(cross)
        for k in range(ns):
            b, q = 100 * k, f"{p}s{k}_"
            ids = r[b + 20].astype(np.int32)
            assert np.array_equal(ids, r[b + 31].astype(np.int32)), "obstacle blocks changed between the normals and the forces"
            n = len(ids)
            npts = r[b + 21].astype(np.int64)
            out[q + "ids"] = ids
            out[q + "npts"] = npts
            out[q + "surf"] = r[b + 22].reshape(-1, 5)
            out[q + "u"], out[q + "v"], out[q + "cmx"], out[q + "cmy"] = r[b + 30]
            out[q + "chi"] = r[b + 32].reshape(n, 8, 8)
            out[q + "udef"] = r[b + 33].reshape(n, 8, 8, 2)
            skin = r[b + 34].reshape(-1, 14)
            copies = skin_copies(blocks, h0, out[p + "vel"], out[p + "pres"],
                                 dict(ids=ids, npts=npts, surf=out[q + "surf"], udef=out[q + "udef"]))
            rest = [c2 for c2 in range(14) if c2 not in SKIN_KEPT]
            assert np.array_equal(copies[:, rest], skin[:, rest]), "a skin column is not the copy it should be"
            out[q + "skin5"] = skin[:, SKIN_KEPT]
            out[q + "acc"] = r[b + 35].reshape(n, 19)
            out[q + "q19"] = r[b + 36]
            out[q + "derived4"] = r[b + 37]
            assert len(out[q + "surf"]) == npts.sum() == len(out[q + "skin5"])
    out["nsteps"] = len(steps)
    np.savez_compressed(OUT, **out)
    print("amrforces", len(steps), "steps;", [len(out[f"c{c}_blocks"]) for c in range(len(steps))], "blocks;",
          [[len(out[f"c{c}_s{k}_ids"]) for k in range(out["nshapes"])] for c in range(len(steps))], "obstacle blocks;",
          [[int(out[f"c{c}_s{k}_npts"].sum()) for k in range(out["nshapes"])] for c in range(len(steps))], "surface points;",
          jumps, "obstacle blocks with surface points and a lab across a level jump;", os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
