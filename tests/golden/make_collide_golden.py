"""Generate tests/golden/amrcollide_lmax8.npz: the reference's own collision model (main.cpp:6705-6943) on its run.sh mesh with
two overlapping fish (tests/golden/ref_collide.cpp).

Run in the build container (needs /root/reference, which does not exist on the GPU box):

    python tests/golden/make_collide_golden.py

ref_collide.cpp includes the unmodified reference main.cpp and is compiled here with the reference's flags (those of
oracle/Makefile) into a temporary directory.  Two placements, two time steps each (one OpenMP thread):
  head  fish head to head: the pair passes every test and the impulse changes (u, v, omega) of both;
  tail  fish tail to tail: the overlap passes the proximity test, projVel <= 0, the motion is unchanged.
Per call: the mesh and per shape the obstacle blocks (ids, chi, dist, udef), (u, v, omega) before and after, centerOfMass, M,
J, length, and the all-reduced 20 N buffer.  load() gives a list of calls.
"""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("CUP2D_REFERENCE", "/root/reference")
LEVEL_MAX, COUNT = 8, 2
OUT = os.path.join(HERE, f"amrcollide_lmax{LEVEL_MAX}.npz")
CONFIGS = (("head", "angle=180 L=0.2 xpos=1.8 ypos=0.8\n angle=0 L=0.2 xpos=1.66 ypos=0.81"),
           ("tail", "angle=0 L=0.2 xpos=1.8 ypos=0.8\n angle=180 L=0.2 xpos=1.66 ypos=0.81"))
SHAPE = ("u", "v", "omega", "cmx", "cmy", "M", "J", "length")


def compile_harness(tmp):
    flags = ["-O3", "-fopenmp", "-std=c++17", "-D_BS_=8", "-include", "cfloat", "-I", os.path.join(ROOT, "oracle", "shim"),
             "-I", REF, "-w"]
    objs = []
    for src in (os.path.join(HERE, "ref_collide.cpp"), os.path.join(ROOT, "oracle", "ref_spmat_cpu.cpp")):
        o = os.path.join(tmp, os.path.basename(src) + ".o")
        subprocess.run(["/usr/bin/g++", *flags, "-c", src, "-o", o], check=True)
        objs.append(o)
    exe = os.path.join(tmp, "ref_collide")
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
    """list of calls; a call is a dict with config, blocks, bpdx, bpdy, h0, sums20 [N, 20], uvw_after [N, 3] and `shapes`, a
    list of per-shape dicts (ids, chi, dist, udef, u, v, omega, center_of_mass, M, J, length)"""
    d = dict(np.load(path))
    out = []
    for c in range(int(d["ncalls"])):
        p = f"c{c}_"
        call = {k[len(p):]: v for k, v in d.items() if k.startswith(p) and "_s" not in k[len(p):]}
        call.update(config=str(d[p + "config"]), bpdx=int(d["bpdx"]), bpdy=int(d["bpdy"]), h0=float(d["h0"]))
        call["shapes"] = []
        for k in range(int(d["nshapes"])):
            q = f"{p}s{k}_"
            s = {key[len(q):]: v for key, v in d.items() if key.startswith(q)}
            s.update(center_of_mass=np.array([float(s.pop("cmx")), float(s.pop("cmy"))]),
                     **{n: float(s[n]) for n in ("u", "v", "omega", "M", "J", "length")})
            call["shapes"].append(s)
        out.append(call)
    return out


def main():
    if not os.path.exists(os.path.join(REF, "main.cpp")):
        sys.exit(f"the reference sources are needed: {REF}/main.cpp")
    out, c = {}, 0
    with tempfile.TemporaryDirectory() as tmp:
        exe = compile_harness(tmp)
        for name, shapes in CONFIGS:
            fout = os.path.join(tmp, f"{name}.bin")
            subprocess.run([exe, str(LEVEL_MAX), str(COUNT), fout, shapes], check=True, stdout=subprocess.DEVNULL,
                           stderr=subprocess.DEVNULL, env=dict(os.environ, OMP_NUM_THREADS="1"))
            calls = records(fout)
            assert len(calls) == COUNT, len(calls)
            for r in calls:
                call, ns, h0, bpdx, bpdy = r[1]
                ns = int(ns)
                out.update(nshapes=ns, h0=h0, bpdx=int(bpdx), bpdy=int(bpdy))
                p = f"c{c}_"
                out[p + "config"] = np.array(name)
                out[p + "step"] = int(call)
                out[p + "blocks"] = r[2].reshape(-1, 3).astype(np.int32)
                out[p + "sums20"] = r[30].reshape(ns, 20)
                out[p + "uvw_after"] = r[31].reshape(ns, 3)
                for k in range(ns):
                    b, q = 100 * k, f"{p}s{k}_"
                    for n, v in zip(SHAPE, r[b + 10]):
                        out[q + n] = v
                    ids = r[b + 20].astype(np.int32)
                    n = len(ids)
                    out[q + "ids"] = ids
                    out[q + "chi"] = r[b + 21].reshape(n, 8, 8)
                    out[q + "dist"] = r[b + 22].reshape(n, 8, 8)
                    out[q + "udef"] = r[b + 23].reshape(n, 8, 8, 2)
                c += 1
    out["ncalls"] = c
    # both branches of the pair loop: an applied impulse (head) and a pair that passes the proximity test without one (tail)
    moved = {str(out[f"c{i}_config"]): [] for i in range(c)}
    for i in range(c):
        before = np.array([[out[f"c{i}_s{k}_{n}"] for n in ("u", "v", "omega")] for k in range(out["nshapes"])])
        s = out[f"c{i}_sums20"]
        near = (s[:, 0] >= 2).all() and (s[:, 10] >= 2).all()
        moved[str(out[f"c{i}_config"])].append((near, not np.array_equal(before, out[f"c{i}_uvw_after"])))
    assert all(near and hit for near, hit in moved["head"]), moved
    assert all(near and not hit for near, hit in moved["tail"]), moved
    np.savez_compressed(OUT, **out)
    print("amrcollide", c, "calls;", [len(out[f"c{i}_blocks"]) for i in range(c)], "blocks;",
          [[len(out[f"c{i}_s{k}_ids"]) for k in range(out["nshapes"])] for i in range(c)], "obstacle blocks; iM",
          [out[f"c{i}_sums20"][:, 0].tolist() for i in range(c)], "; impulse", moved, ";", os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
