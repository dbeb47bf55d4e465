"""Generate tests/golden/amrregrid_lmax8.npz: the reference's own adapt() on its run.sh mesh (tests/golden/ref_aregrid.cpp).

Run in the build container (needs /root/reference, which does not exist on the GPU box):

    python tests/golden/make_regrid_golden.py

ref_aregrid.cpp includes the unmodified reference main.cpp and is compiled here with the reference's flags (those of
oracle/Makefile) into a temporary directory.  Stored, to keep the fixture small: the state before adapt() (mesh, tolerances,
per-block L-inf of the tagging field, vel, pres, chi, tmp — vold and pold are seeded equal to vel and pres), the
{-1,-1,2,2,tensorial} labs of vel and pres of the refined blocks only, the new mesh, and the fields of the new blocks that are
NOT copies of an old block (`new_made` indexes them in the new mesh; every other new block equals the old block with its
(level, i, j)).  load() rebuilds the full arrays of all six transferred fields.
"""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("CUP2D_REFERENCE", "/root/reference")
FIELDS = (("vel", 2), ("vold", 2), ("pres", 1), ("pold", 1), ("chi", 1), ("tmp", 1))
SAME = {"vold": "vel", "pold": "pres"}   # seeded equal: stored once
# levelMax 8: the smallest for which the run.sh fish fit the mesh; Rtol at the 60 % point refines 17 blocks on five levels
LEVEL_MAX, NSTEPS, RQ, CQ = 8, 3, 0.6, 0.1
OUT = os.path.join(HERE, f"amrregrid_lmax{LEVEL_MAX}.npz")


def compile_harness(tmp):
    flags = ["-O3", "-fopenmp", "-std=c++17", "-D_BS_=8", "-include", "cfloat", "-I", os.path.join(ROOT, "oracle", "shim"),
             "-I", REF, "-w"]
    objs = []
    for src in (os.path.join(HERE, "ref_aregrid.cpp"), os.path.join(ROOT, "oracle", "ref_spmat_cpu.cpp")):
        o = os.path.join(tmp, os.path.basename(src) + ".o")
        subprocess.run(["/usr/bin/g++", *flags, "-c", src, "-o", o], check=True)
        objs.append(o)
    exe = os.path.join(tmp, "ref_aregrid")
    subprocess.run(["/usr/bin/g++", "-fopenmp", "-o", exe, *objs], check=True)
    return exe


def records(path):
    a = np.fromfile(path)
    i, rec = 0, {}
    while i < len(a):
        tag, n = int(a[i]), int(a[i + 1])
        rec[tag] = a[i + 2:i + 2 + n]
        i += 2 + n
    return rec


def coverage(blocks, new, bpdx, bpdy):
    """levels on which blocks were refined / compressed, and what the refined blocks touch (8 neighbour positions)"""
    old = {tuple(b): k for k, b in enumerate(blocks.tolist())}
    newset = set(map(tuple, new.tolist()))
    refined = [k for k, (l, i, j) in enumerate(blocks.tolist()) if (l + 1, 2 * i, 2 * j) in newset]
    compressed = [k for k, (l, i, j) in enumerate(blocks.tolist()) if (l - 1, i // 2, j // 2) in newset]
    touch = {"coarser": 0, "finer": 0, "wall": 0}
    for k in refined:
        l, I, J = blocks[k].tolist()
        for x in (-1, 0, 1):
            for y in (-1, 0, 1):
                if (x, y) == (0, 0):
                    continue
                if not (0 <= I + x < bpdx << l and 0 <= J + y < bpdy << l):
                    touch["wall"] += 1
                elif (l, I + x, J + y) not in old:
                    touch["coarser" if (l - 1, (I + x) // 2, (J + y) // 2) in old else "finer"] += 1
    return refined, compressed, touch


def load(path):
    """the fixture with the full new fields rebuilt: dict of arrays"""
    d = dict(np.load(path))
    for a, b in SAME.items():
        d[a], d["new_" + a] = d[b], d["new_" + b]
    old = {tuple(b): k for k, b in enumerate(d["blocks"].tolist())}
    new = d["new_blocks"]
    copied = np.array([old.get(tuple(b), -1) for b in new.tolist()])
    for name, dim in FIELDS:
        full = np.empty((len(new), 8, 8, dim))
        full[copied >= 0] = d[name][copied[copied >= 0]]
        full[d["new_made"]] = d["new_" + name]
        d["new_" + name] = full
    return d


def main():
    if not os.path.exists(os.path.join(REF, "main.cpp")):
        sys.exit(f"the reference sources are needed: {REF}/main.cpp")
    with tempfile.TemporaryDirectory() as tmp:
        exe = compile_harness(tmp)
        fout = os.path.join(tmp, "aregrid.bin")
        subprocess.run([exe, str(LEVEL_MAX), str(NSTEPS), repr(RQ), repr(CQ), fout], check=True, stdout=subprocess.DEVNULL,
                       stderr=subprocess.DEVNULL, env=dict(os.environ, OMP_NUM_THREADS="1"))
        rec = records(fout)
    rtol, ctol, lmax, h0, bpdx, bpdy = rec[10]
    bpdx, bpdy = int(bpdx), int(bpdy)
    blocks = rec[11].reshape(-1, 3).astype(np.int32)
    new = rec[50].reshape(-1, 3).astype(np.int32)
    nb, nn = len(blocks), len(new)
    refined, compressed, touch = coverage(blocks, new, bpdx, bpdy)
    old = {tuple(b) for b in blocks.tolist()}
    made = np.array([q for q, b in enumerate(new.tolist()) if tuple(b) not in old], dtype=np.int32)
    tags_old = {"vel": 12, "vold": 16, "pres": 13, "pold": 17, "chi": 14, "tmp": 18}
    tags_new = {"vel": 51, "vold": 52, "pres": 53, "pold": 54, "chi": 55, "tmp": 56}
    out = dict(rtol=rtol, ctol=ctol, level_max=int(lmax), h0=h0, bpdx=bpdx, bpdy=bpdy, blocks=blocks, block_linf=rec[42],
               new_blocks=new, new_made=made, lab_blocks=np.array(refined, dtype=np.int32),
               lab_vel=rec[24].reshape(nb, 10, 10, 2)[refined], lab_pres=rec[25].reshape(nb, 10, 10, 1)[refined])
    for a, b in SAME.items():
        assert np.array_equal(rec[tags_old[a]], rec[tags_old[b]]) and np.array_equal(rec[tags_new[a]], rec[tags_new[b]])
    for name, dim in FIELDS:
        if name not in SAME:
            out[name] = rec[tags_old[name]].reshape(nb, 8, 8, dim)
            out["new_" + name] = rec[tags_new[name]].reshape(nn, 8, 8, dim)[made]
    np.savez_compressed(OUT, **out)
    levels = sorted(set(blocks[refined, 0].tolist()))
    print("amrregrid", nb, "->", nn, "blocks; refined", len(refined), "on levels", levels, "; compressed", len(compressed), touch,
          ";", os.path.getsize(OUT), "bytes")
    # on this graded mesh nothing can compress (every coarser block touches finer ones, every finest sibling group holds a
    # block of the chi rule): compression is covered by the synthetic meshes of the tests
    assert len(levels) >= 3 and min(touch.values()) > 0


if __name__ == "__main__":
    main()
