"""GPU tests of the reference's multi-level fish loop with every field on the device: oracle/_ref/ref_harness_amrdevice
(oracle/amrdevice.mk, dropin/amr_device_*.inc: ongrid, adapt()'s tagging and in-place regrid, the initial u_def blend,
RK2, the penalisation sums, the collision model, blend, u_def, the pressure section and the forces on one cup2d_amr context)
against the unmodified reference loop (tests/golden/driver_afish_*.npz, recorded from oracle/_ref/ref_afish), and the blend
kernel cup2d_amr_udef_blend against numpy.

They also run on the CPU against the emulated build of the same sources (tests/test_amr_device_loop.py)."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = [pytest.mark.gpu]

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# body state columns of an afish record and the bound each is held to, relative to the quantity's largest magnitude over the run
STATE = ("com_x", "com_y", "orientation", "u", "v", "omega", "M", "J")
STATE_BOUND = 1e-12
FORCE_BOUND = 1e-12


def run_afish(exe, level_max, nsteps, kiter, out, cwd=None, **env):
    env = dict(os.environ, OMP_NUM_THREADS="1", CUP2D_B200_MAX_ITER=str(kiter), CUP2D_B200_AMR_FAST="1", **env)
    subprocess.run([exe, "afish", str(level_max), str(nsteps), str(kiter), str(out)], check=True, stderr=subprocess.DEVNULL,
                   stdout=subprocess.DEVNULL, env=env, timeout=900, cwd=cwd)
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    from make_afish_golden import parse_afish
    return parse_afish(out)


def impulse_steps(bodies):
    """steps at which the collision model changed a velocity: (u, v, omega) before (columns 27-29) != after (30-32)"""
    return [s for s, b in enumerate(bodies) if not np.array_equal(b[:, 27:30], b[:, 30:33])]


def compare(steps, g):
    """per step: mesh identical, dt and the sampled fields within the bounds of the multi-level drop-in test
    (test_gpu_amr.py::test_reference_amr_case_on_the_multi_level_device_path); returns the largest deviations of the body
    state and of each force quantity, relative to that quantity's largest magnitude over the run"""
    ns = int(g["nsteps"])
    assert len(steps) == ns
    ref = np.stack([g[f"bodies_{s}"] for s in range(ns)])
    got = np.stack([r["bodies"] for r in steps])
    for s, r in enumerate(steps):
        assert np.array_equal(r["mesh"], g[f"mesh_{s}"]), s
        assert abs(r["dt"] - g[f"dt_{s}"]) < 1e-14, s
        assert np.abs(r["vel"][g[f"vel_idx_{s}"]] - g[f"vel_{s}"]).max() < 1e-10 * g[f"vel_absmax_{s}"], s
        assert np.abs(r["pres"][g[f"pres_idx_{s}"]] - g[f"pres_{s}"]).max() < 1e-9 * g[f"pres_absmax_{s}"], s
    scale = np.abs(ref).max(axis=0).max(axis=0)
    dev = (np.abs(got - ref).max(axis=0).max(axis=0)) / np.where(scale > 0, scale, 1.0)
    return dev[:8], dev[8:27], ref, got


@pytest.fixture(scope="module")
def exe():
    path = os.path.join(ROOT, "oracle", "_ref", "ref_harness_amrdevice")
    if not os.path.exists(path):
        pytest.skip("oracle/_ref/ref_harness_amrdevice not built (make -C oracle -f amrdevice.mk: needs the reference sources)")
    return path


@pytest.mark.parametrize("fixture", ["lmax8_k8", "collide_lmax8_k8"])
def test_reference_amr_fish_loop_with_every_field_on_the_device(golden_dir, tmp_path, exe, fixture):
    """(a) the run.sh case, 9 steps across the regrid of step 7 (278 -> 281 blocks); (b) two fish overlapping head to head, where
    the collision impulse fires from step 0 on.  Mesh identical, dt and fields within the drop-in bounds, the glue moves no field
    byte after the initial upload, the impulse fires at the same steps as in the reference.
    Body state (centre of mass, orientation, u, v, omega, M, J) and each of the 19 force quantities within 1e-12 of the
    quantity's largest magnitude over the run.  Measured on an H100: 9.4e-15 (u) and 1.8e-14 (forces) at most, on the CPU
    emulation 6e-14.  Not bitwise: the penalisation sums and ongrid()'s moments are added per block rather than in the
    reference's OpenMP order, and the chi of blocks whose lab crosses a level jump comes from the plan's ghost rows; u, v and
    omega then come out of a 3x3 solve on those sums and feed the forces.  The bound keeps a factor 50 over the measurement."""
    g = np.load(os.path.join(golden_dir, f"driver_afish_{fixture}.npz"))
    steps = run_afish(exe, int(g["level_max"]), int(g["nsteps"]), int(g["kiter"]), tmp_path / "afish.bin",
                      **({"CUP2D_REF_SHAPES": str(g["shapes"])} if str(g["shapes"]) else {}))
    dstate, dforce, ref, got = compare(steps, g)
    print(f"{fixture}: body state", dict(zip(STATE, dstate)), "forces max", dforce.max(), "argmax", int(dforce.argmax()))
    assert all(r["field_bytes"] == 0 for r in steps)
    assert dstate.max() < STATE_BOUND, dict(zip(STATE, dstate))
    assert dforce.max() < FORCE_BOUND, dforce
    assert impulse_steps(got) == impulse_steps(ref)
    if fixture.startswith("collide"):
        assert impulse_steps(ref)[:1] == [0]
    else:
        assert impulse_steps(ref) == [] and len(steps[0]["mesh"]) == 278 and len(steps[-1]["mesh"]) == 281


def test_reference_amr_fish_loop_dump_from_the_device(golden_dir, tmp_path, exe):
    """-tdump > 0: dump() at the start of a step writes vel.<step>.attr.raw from the device (cup2d_amr_dump); it holds (u, v, 0)
    of the velocity the previous step ended with, narrowed to float32, which is what the afish record of that step holds in
    float64"""
    steps = run_afish(exe, 8, 4, 8, tmp_path / "afish.bin", cwd=tmp_path, CUP2D_REF_TDUMP="0.04")
    dumped = sorted(int(f.split(".")[1]) for f in os.listdir(tmp_path) if f.endswith(".attr.raw"))
    assert len([s for s in dumped if s >= 1]) >= 1, dumped
    for s in dumped:
        if s == 0:
            continue
        attr = np.fromfile(tmp_path / f"vel.{s:08d}.attr.raw", dtype=np.float32).reshape(-1, 3)
        vel = steps[s - 1]["vel"].reshape(-1, 2)
        assert np.array_equal(attr[:, :2], vel.astype(np.float32)) and not attr[:, 2].any(), s


def test_amr_udef_blend_bitwise_against_numpy(golden_dir):
    """cup2d_amr_udef_blend: vel = vel (1 - chi) + tmpV chi (main.cpp:6566-6575) on the run.sh mesh, bit for bit"""
    from cup2d_b200.amr import AmrSimulation
    d = np.load(os.path.join(golden_dir, "amrlab_lmax8.npz"))
    nb = len(d["blocks"])
    rng = np.random.default_rng(11)
    vel, tmpv = rng.uniform(-1, 1, (nb, 8, 8, 2)), rng.uniform(-1, 1, (nb, 8, 8, 2))
    chi = rng.uniform(0, 1, (nb, 8, 8, 1))
    chi[rng.uniform(0, 1, chi.shape) < 0.3] = 0.0
    chi[rng.uniform(0, 1, chi.shape) < 0.2] = 1.0
    sim = AmrSimulation(d["blocks"], int(d["bpdx"]), int(d["bpdy"]), float(d["h0"]), float(d["nu"]))
    try:
        sim.upload("vel", vel)
        sim.upload("tmpV", tmpv)
        sim.upload("chi", chi)
        sim.udef_blend()
        got = sim.download("vel")
    finally:
        sim.close()
    want = vel * (1 - chi) + tmpv * chi
    assert np.array_equal(got, want)
