"""Generate tests/golden/amrongrid_lmax8.npz: the reference's own ongrid() on its run.sh mesh (tests/golden/ref_ongrid.cpp).

Run in the build container (needs /root/reference, which does not exist on the GPU box):

    python tests/golden/make_ongrid_golden.py

ref_ongrid.cpp includes the unmodified reference main.cpp and is compiled here with the reference's flags (those of
oracle/Makefile) into a temporary directory.  Recorded: the ongrid() calls of the first time steps (each on the mesh adapt()
left for that step), two fish.  Per call: the mesh, the chi and tmp fields after PutChiOnGrid, and per shape the midline state
ongrid() rasterises (main.cpp:4208), the obstacle blocks with dist, chi, u_def before and after the rigid-motion removal, the
per-block Mass / COM partials, com[3], the seven sums and the new centre of mass, M and J.  load() gives a list of calls.
"""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("CUP2D_REFERENCE", "/root/reference")
# levelMax 8: the 7-level mesh of the other AMR fixtures.  The setup makes levelMax + 1 ongrid() calls (main.cpp:6542-6546);
# FIRST skips them, so the recorded calls are those of time steps 0, 1, ... (dt > 0: the bodies have moved)
LEVEL_MAX, FIRST, COUNT = 8, 9, 2
OUT = os.path.join(HERE, f"amrongrid_lmax{LEVEL_MAX}.npz")
MIDLINE = ("rX", "rY", "norX", "norY", "vX", "vY", "vNorX", "vNorY", "width")


def compile_harness(tmp):
    flags = ["-O3", "-fopenmp", "-std=c++17", "-D_BS_=8", "-include", "cfloat", "-I", os.path.join(ROOT, "oracle", "shim"),
             "-I", REF, "-w"]
    objs = []
    for src in (os.path.join(HERE, "ref_ongrid.cpp"), os.path.join(ROOT, "oracle", "ref_spmat_cpu.cpp")):
        o = os.path.join(tmp, os.path.basename(src) + ".o")
        subprocess.run(["/usr/bin/g++", *flags, "-c", src, "-o", o], check=True)
        objs.append(o)
    exe = os.path.join(tmp, "ref_ongrid")
    subprocess.run(["/usr/bin/g++", "-fopenmp", "-o", exe, *objs], check=True)
    return exe


def records(path):
    """the record stream split into calls: list of {tag: array}"""
    a = np.fromfile(path)
    i, calls = 0, []
    while i < len(a):
        tag, n = int(a[i]), int(a[i + 1])
        if tag == 1:
            calls.append({})
        calls[-1][tag] = a[i + 2:i + 2 + n]
        i += 2 + n
    return calls


def load(path):
    """list of calls; a call is a dict with blocks, bpdx, bpdy, h0, extent, chi, tmp and `shapes`, a list of per-shape dicts"""
    d = dict(np.load(path))
    out = []
    for c in range(int(d["ncalls"])):
        p = f"c{c}_"
        call = {k[len(p):]: v for k, v in d.items() if k.startswith(p) and "_s" not in k[len(p):]}
        call.update(bpdx=int(d["bpdx"]), bpdy=int(d["bpdy"]), h0=float(d["h0"]), extent=d["extent"])
        call["shapes"] = []
        for k in range(int(d["nshapes"])):
            q = f"{p}s{k}_"
            call["shapes"].append({key[len(q):]: v for key, v in d.items() if key.startswith(q)})
        out.append(call)
    return out


def main():
    if not os.path.exists(os.path.join(REF, "main.cpp")):
        sys.exit(f"the reference sources are needed: {REF}/main.cpp")
    with tempfile.TemporaryDirectory() as tmp:
        exe = compile_harness(tmp)
        fout = os.path.join(tmp, "ongrid.bin")
        subprocess.run([exe, str(LEVEL_MAX), str(FIRST), str(COUNT), fout], check=True, stdout=subprocess.DEVNULL,
                       stderr=subprocess.DEVNULL, env=dict(os.environ, OMP_NUM_THREADS="1"))
        calls = records(fout)
    assert len(calls) == COUNT
    head = calls[0][1]
    ns = int(head[1])
    out = dict(ncalls=COUNT, nshapes=ns, h0=head[2], extent=head[3:5].copy(), bpdx=int(head[5]), bpdy=int(head[6]))
    for c, r in enumerate(calls):
        p = f"c{c}_"
        blocks = r[2].reshape(-1, 3).astype(np.int32)
        nb = len(blocks)
        out[p + "blocks"] = blocks
        out[p + "chi"] = r[3].reshape(nb, 8, 8)
        out[p + "tmp"] = r[4].reshape(nb, 8, 8)
        for k in range(ns):
            b, q = 100 * k, f"{p}s{k}_"
            nm, cx, cy, ang, gx, gy = r[b + 10]
            out[q + "center"], out[q + "orientation"], out[q + "center_of_mass"] = np.array([cx, cy]), ang, np.array([gx, gy])
            for m, name in enumerate(MIDLINE):
                out[q + name] = r[b + 11 + m]
                assert len(r[b + 11 + m]) == int(nm)
            ids = r[b + 20].astype(np.int32)
            n = len(ids)
            out[q + "ids"] = ids
            out[q + "dist"] = r[b + 21].reshape(n, 8, 8)
            out[q + "chi"] = r[b + 22].reshape(n, 8, 8)
            out[q + "udef_pre"] = r[b + 23].reshape(n, 8, 8, 2)
            out[q + "mass_com"] = r[b + 24].reshape(n, 3)
            out[q + "com3"] = r[b + 25]
            out[q + "sums7"] = r[b + 26]
            out[q + "udef"] = r[b + 27].reshape(n, 8, 8, 2)
            gx1, gy1, M, J = r[b + 28]
            out[q + "new_center_of_mass"], out[q + "M"], out[q + "J"] = np.array([gx1, gy1]), M, J
    np.savez_compressed(OUT, **out)
    print("amrongrid", COUNT, "calls;", [len(out[f"c{c}_blocks"]) for c in range(COUNT)], "blocks;",
          [[len(out[f"c{c}_s{k}_ids"]) for k in range(ns)] for c in range(COUNT)], "obstacle blocks; Nm",
          len(out["c0_s0_rX"]), ";", os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
