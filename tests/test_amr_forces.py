"""CPU tests of the surface normals and force diagnostics on multi-level meshes: the oracle (tests/amr_forces_oracle.py)
against the reference's own ComputeSurfaceNormals and KernelComputeForces on its run.sh mesh (tests/golden/amrforces_lmax8.npz),
the plan's lab kind 6 against the reference's VectorLab, and the device code (tests/test_gpu_amr_forces.py) on the emulated
library."""
import os
import subprocess
import sys

import numpy as np
import pytest

import amr_forces_oracle as fo

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def steps(golden_dir):
    sys.path.insert(0, golden_dir)
    import make_forces_golden
    return make_forces_golden.load(os.path.join(golden_dir, "amrforces_lmax8.npz"))


def test_oracle_equals_the_reference_bit_for_bit(steps):
    """point lists, skin arrays, per-block accumulators, the 19-value buffer and the derived four, every bit"""
    for st in steps:
        pts = fo.normals(st["blocks"], st["bpdx"], st["bpdy"], st["h0"], st["chi_n"], st["tmp"], [s["ids"] for s in st["shapes"]])
        for s, P in zip(st["shapes"], pts):
            assert np.array_equal([len(b) for b in P], s["npts"])
            assert np.array_equal(np.array([p for b in P for p in b]).reshape(-1, 5), s["surf"])
        res = fo.forces(st["blocks"], st["bpdx"], st["bpdy"], st["h0"], st["nu"], st["vel"], st["pres"], st["chi_n"],
                        st["shapes"], pts)
        for s, r in zip(st["shapes"], res):
            for k in ("skin", "acc", "q19", "derived4"):
                assert np.array_equal(r[k], s[k]), k


def test_fixture_covers_the_reference_details(steps):
    """the fixture exercises what the restatement has to get right: corner-ghost points, level jumps, every derivative branch"""
    st = steps[0]
    # points at the cells that read a corner ghost of the normals' lab (the reference's unwritten lab memory)
    cells = {(int(p[0]), int(p[1])) for s in st["shapes"] for p in s["surf"]}
    assert {(0, 0), (7, 0), (0, 7)} <= cells
    nocorner = fo.normals(st["blocks"], st["bpdx"], st["bpdy"], st["h0"], st["chi_n"], st["tmp"],
                          [s["ids"] for s in st["shapes"]], corner=(np.nan, np.nan))
    assert sum(len(b) for P in nocorner for b in P) < sum(len(s["surf"]) for s in st["shapes"])
    # u, v of the shapes are not zero (vel_unit is taken), and both thrust and drag are present
    for s in st["shapes"]:
        assert s["u"] != 0 and s["q19"][16] > 0 and s["q19"][6] > 0
        assert (s["acc"][:, 10] < 0).any() and (s["acc"][:, 17] < 0).any()   # PoutBnd, defPowerBnd: min(0, .) taken


def test_plan_kind6_reproduces_the_reference_vector_lab(steps):
    """stencil kind 6 = KernelComputeForces's {-4,-4,5,5,tensorial} velocity lab (free-slip walls): the tables applied to the
    recorded vel give the reference's VectorLab of every obstacle block, to rounding (the criterion of test_amr_plan.py)"""
    from cup2d_b200.amr import AmrPlan
    st = steps[0]
    nb = len(st["blocks"])
    plan = AmrPlan(np.ascontiguousarray(st["blocks"], dtype=np.int32), st["bpdx"], st["bpdy"])
    rp, sb, sc, w = plan.stencil(6)
    assert len(rp) == nb * 512 + 1 and (rp[1:] > rp[:-1]).all()       # tensorial: every lab cell has sources
    vals = w * st["vel"].reshape(nb, 128)[sb, sc]
    lab = np.add.reduceat(vals, rp[:-1]).reshape(nb, 16, 16, 2)[st["lab_ids"]]
    want = st["lab_vel"]
    assert np.abs(lab - want).max() < 1e-13 * np.abs(want).max()
    assert np.array_equal(lab[:, 4:12, 4:12], st["vel"][st["lab_ids"]])
    # the compact ghost rows of kind 6 are the full rows of the irregular blocks
    grp, dst, gsb, gsc, gw = plan.ghosts(6)
    irr = plan.irregular()
    full = np.add.reduceat(vals, rp[:-1])
    ghost = np.add.reduceat(gw * st["vel"].reshape(nb, 128)[gsb, gsc], grp[:-1]) if len(gw) else np.zeros(0)
    rows = irr[dst // 512].astype(np.int64) * 512 + dst % 512
    assert np.abs(ghost - full[rows]).max() < 1e-13 * np.abs(want).max()
    assert plan.stats(6)["fallbacks"] == 0
    plan.close()


def test_device_forces_on_the_emulated_library():
    """tests/test_gpu_amr_forces.py on a g++ build of the product sources (tests/host_emu/build.py build_full)"""
    sys.path.insert(0, os.path.join(HERE, "host_emu"))
    import build
    lib = build.build_full()
    env = dict(os.environ, CUP2D_B200_LIB=lib)
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(HERE, "test_gpu_amr_forces.py"), "-m", "gpu", "-q",
                        "-p", "no:cacheprovider"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env,
                       timeout=3000, cwd=ROOT)
    tail = r.stdout[-2000:]
    assert r.returncode == 0 and " passed" in tail and "failed" not in tail and "skipped" not in tail, tail


sanitizers = pytest.mark.skipif(os.environ.get("CUP2D_TEST_SANITIZERS") != "1", reason="sanitizer builds are opt-in: CUP2D_TEST_SANITIZERS=1")


@sanitizers
@pytest.mark.parametrize("sanitize", ["thread", "address,alignment,bounds"])
def test_forces_under_sanitizers(sanitize):
    """tests/host_emu/forces_driver.cpp (an ongrid body across a level jump, surface and two forces calls) linked against the
    emulated product sources built with ThreadSanitizer / AddressSanitizer: no report, no NaN from never-written memory"""
    sys.path.insert(0, os.path.join(HERE, "host_emu"))
    import build
    build.build_full()
    tag = "tsan" if sanitize == "thread" else "asan"
    srcs = [os.path.join(build.FULL, f) for f in sorted(os.listdir(build.FULL)) if f.endswith(".cpp")]
    exe = os.path.join(build.FULL, f"forces_{tag}_driver")
    try:
        build._compile_link(["-O1", "-g", "-std=c++20", "-pthread", f"-fsanitize={sanitize}",
                             *([] if sanitize == "thread" else ["-fno-sanitize-recover=all"]), "-w", "-DEMU_ALL_COOP",
                             "-I", build.FULL, "-I", os.path.join(HERE, "host_emu")],
                            [os.path.join(HERE, "host_emu", "forces_driver.cpp"), *srcs], exe,
                            os.path.join(build.FULL, f"obj_forces_{tag}"))
    except subprocess.CalledProcessError:
        pytest.skip(f"the {sanitize} sanitizer runtime is not available to g++ on this box")
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0", ASAN_OPTIONS="detect_leaks=0")
    r = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=3000, env=env)
    assert r.returncode == 0, r.stdout[-3000:]
    assert "Sanitizer" not in r.stdout and "runtime error" not in r.stdout, r.stdout[-3000:]
    assert r.stdout.count("forces call") == 2 and "nan" not in r.stdout.lower(), r.stdout[-3000:]
