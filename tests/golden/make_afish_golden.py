"""Generate the golden records of the reference's multi-level fish loop that the device-form tests compare against.

    python tests/golden/make_afish_golden.py     # oracle/_ref/ref_afish: the UNMODIFIED reference, no GPU needed

oracle/_ref/ref_afish is built by `make -C oracle -f amrdevice.mk afish` from the reference sources (oracle/ref_afish.cpp
documents the record).  One OpenMP thread and a fixed number of Poisson iterations, so that a record regenerates
bit-identically.  Dt, the mesh, the body state, the forces and the velocities around the collision model are kept in full, the
fields at a fixed, seeded sample of entries (`*_idx`) plus each field's full-field max |.| (`*_absmax`) for the relative
bounds of the tests.
"""
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.path.join(ROOT, "oracle", "_ref")
AFISH_SHAPE = 33   # per shape: centerOfMass[2], orientation, u, v, omega, M, J, 19 forces, (u, v, omega) before / after collisions
FORCES = ("circulation", "perimeter", "forcex", "forcex_P", "forcex_V", "torque_P", "drag", "lift", "Pout", "PoutNew", "PoutBnd",
          "torque", "forcey", "forcey_P", "forcey_V", "torque_V", "thrust", "defPowerBnd", "defPower")
COLLIDE_SHAPES = "angle=180 L=0.2 xpos=1.8 ypos=0.8\n angle=0 L=0.2 xpos=1.66 ypos=0.81"   # head to head, overlapping


def sample(n, m, seed):
    return np.sort(np.random.default_rng(seed).choice(n, m, replace=False)) if m < n else np.arange(n)


def parse_afish(path):
    """`afish` records: per step a dict of dt, field_bytes, wall, time, mesh, vel, pres, bodies [S, 33]"""
    a, i, out = np.fromfile(path), 0, []
    while i < len(a):
        dt, nb, ns, nbytes, wall, time = a[i:i + 6]
        nb, ns = int(nb), int(ns)
        i += 6
        mesh = a[i:i + 3 * nb].reshape(nb, 3).astype(np.int32)
        i += 3 * nb
        vel, pres = a[i:i + 128 * nb], a[i + 128 * nb:i + 192 * nb]
        i += 192 * nb
        bodies = a[i:i + AFISH_SHAPE * ns].reshape(ns, AFISH_SHAPE)
        i += AFISH_SHAPE * ns
        out.append(dict(dt=dt, field_bytes=nbytes, wall=wall, time=time, mesh=mesh, vel=vel, pres=pres, bodies=bodies))
    return out


def gen_afish(tmp, level_max, nsteps, kiter, name, shapes=None):
    """the run.sh case (or `shapes`): per step dt, mesh, vel and pres blocks (sampled), body state, forces and the velocities
    before / after the collision model, in full"""
    out = os.path.join(tmp, "afish.bin")
    env = dict(os.environ, OMP_NUM_THREADS="1", **({"CUP2D_REF_SHAPES": shapes} if shapes else {}))
    subprocess.run([os.path.join(REF, "ref_afish"), "afish", str(level_max), str(nsteps), str(kiter), out], check=True,
                   stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL, env=env)
    rec = {"level_max": level_max, "kiter": kiter, "nsteps": nsteps, "shapes": shapes or ""}
    for s, r in enumerate(parse_afish(out)):
        iv, ip = sample(len(r["vel"]), 4096, 30 + s), sample(len(r["pres"]), 2048, 40 + s)
        rec.update({f"dt_{s}": r["dt"], f"time_{s}": r["time"], f"mesh_{s}": r["mesh"], f"vel_{s}": r["vel"][iv],
                    f"vel_idx_{s}": iv, f"pres_{s}": r["pres"][ip], f"pres_idx_{s}": ip,
                    f"vel_absmax_{s}": np.abs(r["vel"]).max(), f"pres_absmax_{s}": np.abs(r["pres"]).max(),
                    f"bodies_{s}": r["bodies"]})
    np.savez_compressed(os.path.join(HERE, f"driver_afish_{name}.npz"), **rec)


if __name__ == "__main__":
    with tempfile.TemporaryDirectory() as tmp:
        gen_afish(tmp, 8, 9, 8, "lmax8_k8")                          # test_gpu_amr_device_loop.py: (a) the run.sh case
        gen_afish(tmp, 8, 6, 8, "collide_lmax8_k8", COLLIDE_SHAPES)  # ... (b) a head-to-head collision
        gen_afish(tmp, 8, 3, 5, "lmax8_k5")                          # test_amr_device_loop.py: a prefix of (a), emulated
