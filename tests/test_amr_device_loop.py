"""CPU tests of the reference's multi-level fish loop with every field on the device (tests/test_gpu_amr_device_loop.py) on the
emulated library (tests/host_emu/build.py build_full): the blend kernel against numpy, and oracle/_ref/ref_harness_amrdevice
linked against the emulation on a 3-step prefix of the run.sh case (tests/golden/driver_afish_lmax8_k5.npz)."""
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def emulated_library():
    sys.path.insert(0, os.path.join(HERE, "host_emu"))
    import build
    return build.build_full()


def test_udef_blend_on_the_emulated_library(emulated_library):
    """tests/test_gpu_amr_device_loop.py::test_amr_udef_blend_bitwise_against_numpy on the emulated library"""
    env = dict(os.environ, CUP2D_B200_LIB=emulated_library)
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(HERE, "test_gpu_amr_device_loop.py"), "-m", "gpu", "-q",
                        "-k", "udef_blend", "-p", "no:cacheprovider"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                       env=env, timeout=900, cwd=ROOT)
    tail = r.stdout[-2000:]
    assert r.returncode == 0 and "1 passed" in tail and "failed" not in tail and "skipped" not in tail, tail


def test_reference_amr_fish_loop_on_the_device_path_emulated(emulated_library, golden_dir, tmp_path):
    """the device form of the run.sh case linked against the emulated library, 3 steps against the unmodified reference: mesh
    identical, dt within 1e-15, velocity within 1e-12 and pressure within 1e-11 of their largest magnitude, no field byte moved
    after the initial upload, body state and forces within the bounds of the GPU test (measured here: 6e-14 at most)"""
    if not os.path.exists("/root/reference/main.cpp"):
        pytest.skip("needs the reference sources to build the patched driver (build container only)")
    emu_dir = os.path.dirname(emulated_library)
    subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "-f", "amrdevice.mk", "ref_amrdevice", f"LIBDIR={emu_dir}", "LIBNAME=cup2d_emu",
                    "AMRDEVICE=ref_harness_amrdevice_emu", f"RPATH={emu_dir}"], check=True, stdout=subprocess.DEVNULL)
    sys.path.insert(0, HERE)
    import test_gpu_amr_device_loop as dl
    g = np.load(os.path.join(golden_dir, "driver_afish_lmax8_k5.npz"))
    ns = int(g["nsteps"])
    steps = dl.run_afish(os.path.join(ROOT, "oracle", "_ref", "ref_harness_amrdevice_emu"), int(g["level_max"]), ns,
                         int(g["kiter"]), tmp_path / "afish.bin")
    assert len(steps) == ns == 3
    for s, r in enumerate(steps):
        assert np.array_equal(r["mesh"], g[f"mesh_{s}"]) and abs(r["dt"] - g[f"dt_{s}"]) < 1e-15
        assert np.abs(r["vel"][g[f"vel_idx_{s}"]] - g[f"vel_{s}"]).max() < 1e-12 * g[f"vel_absmax_{s}"]
        assert np.abs(r["pres"][g[f"pres_idx_{s}"]] - g[f"pres_{s}"]).max() < 1e-11 * g[f"pres_absmax_{s}"]
        assert r["field_bytes"] == 0
    dstate, dforce, ref, got = dl.compare(steps, g)
    assert dstate.max() < dl.STATE_BOUND and dforce.max() < dl.FORCE_BOUND, (dstate, dforce)
    assert dl.impulse_steps(got) == dl.impulse_steps(ref) == []
