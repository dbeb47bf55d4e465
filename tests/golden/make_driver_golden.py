"""Generate the golden records of the reference's own time loops that the drop-in tests compare against.

    python tests/golden/make_driver_golden.py cpu    # oracle/_ref/ref_harness: no GPU needed
    python tests/golden/make_driver_golden.py gpu    # oracle/_ref/ref_harness_gpu: the reference's cuda.cu, needs a GPU

Both binaries are the UNMODIFIED reference built by `make -C oracle all` (see oracle/Makefile).  One OpenMP thread, so that
a record regenerates bit-identically.  Records larger than the fixture budget keep dt, the mesh and the body state in full
and the fields at a fixed, seeded sample of entries (`*_idx`), plus each field's full-field max |.| (`*_absmax`) for the
relative bounds of the tests.
"""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.path.join(ROOT, "oracle", "_ref")
SHAPES = "angle=0 L=0.8 xpos=0.52 ypos=0.44\n angle=175 L=0.8 xpos=0.47 ypos=0.56"   # two interacting fish (fsteps)


def run(exe, *args, **env):
    subprocess.run([os.path.join(REF, exe), *map(str, args)], check=True, stdout=subprocess.DEVNULL,
                   stderr=subprocess.DEVNULL, env=dict(os.environ, OMP_NUM_THREADS="1", **env))


def sample(n, m, seed):
    return np.sort(np.random.default_rng(seed).choice(n, m, replace=False)) if m < n else np.arange(n)


def make_fields(N, seed):
    """tests/test_gpu_parity.py:make_fields (kind 'tg'): u, v, p"""
    rng = np.random.default_rng(seed)
    x = (np.arange(N) + 0.5) / N
    X, Y = np.meshgrid(x, x)
    u = np.sin(2 * np.pi * X) * np.cos(2 * np.pi * Y) + 0.05 * rng.uniform(-1, 1, (N, N))
    v = -np.cos(2 * np.pi * X) * np.sin(2 * np.pi * Y) + 0.05 * rng.uniform(-1, 1, (N, N))
    p = np.cos(2 * np.pi * X) * np.cos(2 * np.pi * Y)
    return u, v, p


def gen_fsteps(tmp, L, nsteps, kiter):
    """two fish, uniform level-L grid: per step dt, u v p (sampled), centre of mass, u, v, omega of both fish"""
    out = os.path.join(tmp, "fsteps.bin")
    run("ref_harness", "fsteps", L, nsteps, kiter, out, CUP2D_REF_SHAPES=SHAPES)
    N = 8 << L
    a = np.fromfile(out).reshape(nsteps, 1 + 3 * N * N + 10)
    idx = sample(3 * N * N, 8192, 1)
    fields = a[:, 1:-10]
    np.savez_compressed(os.path.join(HERE, f"driver_fsteps_L{L}_k{kiter}.npz"), L=L, kiter=kiter, dt=a[:, 0],
                        fields=fields[:, idx], fields_idx=idx, bodies=a[:, -10:],
                        u_absmax=np.abs(fields[:, :N * N]).max(axis=1))


def parse_asteps(path):
    a, i, out = np.fromfile(path), 0, []
    while i < len(a):
        dt, nb = a[i], int(a[i + 1])
        i += 2
        mesh = a[i:i + 3 * nb].reshape(nb, 3).astype(np.int32)
        i += 3 * nb
        out.append((dt, mesh, a[i:i + 128 * nb], a[i + 128 * nb:i + 192 * nb]))
        i += 192 * nb
    return out


def gen_asteps(tmp, level_max, nsteps, kiter):
    """the run.sh case (2 fish, regridding): per step dt, mesh, vel and pres blocks (sampled)"""
    out = os.path.join(tmp, "asteps.bin")
    run("ref_harness", "asteps", level_max, nsteps, kiter, out)
    rec = {"level_max": level_max, "kiter": kiter, "nsteps": nsteps}
    for s, (dt, mesh, vel, pres) in enumerate(parse_asteps(out)):
        iv, ip = sample(len(vel), 4096, 10 + s), sample(len(pres), 2048, 20 + s)
        rec.update({f"dt_{s}": dt, f"mesh_{s}": mesh, f"vel_{s}": vel[iv], f"vel_idx_{s}": iv, f"pres_{s}": pres[ip],
                    f"pres_idx_{s}": ip, f"vel_absmax_{s}": np.abs(vel).max(), f"pres_absmax_{s}": np.abs(pres).max()})
    np.savez_compressed(os.path.join(HERE, f"driver_asteps_lmax{level_max}_k{kiter}.npz"), **rec)


def gen_gpu_steps(tmp, L, seed, nsteps, kiter):
    """the reference's own loop with its own GPU solver (cuda.cu): dt, u, v, p per step on make_fields(N, seed)"""
    N = 8 << L
    u, v, p = make_fields(N, seed)
    z = np.zeros((N, N))
    fin, fout = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bin")
    np.concatenate([a.ravel() for a in (u, v, p, z, z, z)]).tofile(fin)
    run("ref_harness_gpu", "steps", L, "1e-3", "0.5", nsteps, kiter, fin, fout)
    a = np.fromfile(fout).reshape(nsteps, 1 + 5 * N * N)
    f = a[:, 1:].reshape(nsteps, 5, N, N)
    np.savez_compressed(os.path.join(HERE, f"driver_gpu_steps_L{L}.npz"), L=L, seed=seed, kiter=kiter, dt=a[:, 0],
                        u=f[:, 0], v=f[:, 1], p=f[:, 2])


def gen_gpu_amr(tmp, level_max, nsteps, kiter):
    """the run.sh case with the reference's cuda.cu: per step dt, mesh, Poisson right-hand side b and solution x"""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from ref_gpu_compare_amr import read_records
    out = os.path.join(tmp, "amr.bin")
    run("ref_harness_gpu", "amr", level_max, nsteps, kiter, out)
    rec = {"level_max": level_max, "kiter": kiter, "nsteps": nsteps}
    for s, r in enumerate(read_records(out)):
        rec.update({f"dt_{s}": r["dt"], f"lij_{s}": r["lij"], f"b_{s}": r["b"], f"x_{s}": r["x"]})
    np.savez_compressed(os.path.join(HERE, f"driver_gpu_amr_lmax{level_max}.npz"), **rec)


if __name__ == "__main__":
    with tempfile.TemporaryDirectory() as tmp:
        if sys.argv[1] == "cpu":
            gen_fsteps(tmp, 4, 4, 8)       # test_gpu_parity.py: resident loop with bodies
            gen_fsteps(tmp, 4, 4, 5)       # test_full_emulation.py: the same on the emulated library
            gen_asteps(tmp, 8, 6, 8)       # test_gpu_amr.py: run.sh case on the multi-level device path
            gen_asteps(tmp, 8, 3, 5)       # test_full_emulation.py: the same on the emulated library
        else:
            gen_gpu_steps(tmp, 3, 77, 1, 1000)   # test_gpu_parity.py: the LocalSpMatDnVec adapter against cuda.cu
            gen_gpu_amr(tmp, 8, 2, 1000)         # test_gpu_parity.py: run.sh case through the adapter against cuda.cu
