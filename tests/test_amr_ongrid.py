"""CPU tests of ongrid() on multi-level meshes: the oracle (tests/amr_body_oracle.py) against the reference's own ongrid() on its
run.sh mesh (tests/golden/amrongrid_lmax8.npz), and the device code (tests/test_gpu_amr_ongrid.py) on the emulated library."""
import os
import subprocess
import sys

import numpy as np
import pytest

import amr_body_oracle as bo

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
FIELDS = ("ids", "dist", "chi", "udef_pre", "mass_com", "com3", "sums7", "new_center_of_mass", "udef")


@pytest.fixture(scope="module")
def calls(golden_dir):
    sys.path.insert(0, golden_dir)
    import make_ongrid_golden
    return make_ongrid_golden.load(os.path.join(golden_dir, "amrongrid_lmax8.npz"))


def test_oracle_equals_the_reference_bit_for_bit(calls):
    for c in calls:
        bodies = [{**{n: s[n] for n in bo.MIDLINE}, "center": s["center"], "orientation": s["orientation"],
                   "center_of_mass": s["center_of_mass"]} for s in c["shapes"]]
        r = bo.ongrid(c["blocks"], c["bpdx"], c["bpdy"], c["h0"], bodies)
        assert np.array_equal(r["tmp"], c["tmp"]) and np.array_equal(r["chi"], c["chi"])
        for got, want in zip(r["shapes"], c["shapes"]):
            for n in FIELDS:
                assert np.array_equal(got[n], want[n]), n
            assert got["out10"][5] == want["M"] and got["out10"][6] == want["J"]


def test_synthetic_bodies_are_valid_midlines():
    b = bo.synthetic_body((0.5, 0.5), 0.2, 161, 0.4)
    assert all(len(b[n]) == 161 for n in bo.MIDLINE)
    assert (b["width"] > 0).all()
    assert np.allclose(np.hypot(b["norX"], b["norY"]), 1.0)


def test_device_ongrid_on_the_emulated_library():
    """tests/test_gpu_amr_ongrid.py on a g++ build of the product sources (tests/host_emu/build.py build_full)"""
    sys.path.insert(0, os.path.join(HERE, "host_emu"))
    import build
    lib = build.build_full()
    env = dict(os.environ, CUP2D_B200_LIB=lib)
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(HERE, "test_gpu_amr_ongrid.py"), "-m", "gpu", "-q",
                        "-p", "no:cacheprovider"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env,
                       timeout=1800, cwd=ROOT)
    tail = r.stdout[-2000:]
    assert r.returncode == 0 and " passed" in tail and "failed" not in tail and "skipped" not in tail, tail


sanitizers = pytest.mark.skipif(os.environ.get("CUP2D_TEST_SANITIZERS") != "1", reason="sanitizer builds are opt-in: CUP2D_TEST_SANITIZERS=1")


@sanitizers
@pytest.mark.parametrize("sanitize", ["thread", "address,alignment,bounds"])
def test_ongrid_under_sanitizers(sanitize):
    """tests/host_emu/ongrid_driver.cpp (two overlapping bodies across a level jump, two calls) linked against the emulated
    product sources built with ThreadSanitizer / AddressSanitizer: no report, no NaN from never-written memory"""
    sys.path.insert(0, os.path.join(HERE, "host_emu"))
    import build
    build.build_full()
    tag = "tsan" if sanitize == "thread" else "asan"
    srcs = [os.path.join(build.FULL, f) for f in sorted(os.listdir(build.FULL)) if f.endswith(".cpp")]
    exe = os.path.join(build.FULL, f"ongrid_{tag}_driver")
    try:
        build._compile_link(["-O1", "-g", "-std=c++20", "-pthread", f"-fsanitize={sanitize}",
                             *([] if sanitize == "thread" else ["-fno-sanitize-recover=all"]), "-w", "-DEMU_ALL_COOP",
                             "-I", build.FULL, "-I", os.path.join(HERE, "host_emu")],
                            [os.path.join(HERE, "host_emu", "ongrid_driver.cpp"), *srcs], exe,
                            os.path.join(build.FULL, f"obj_ongrid_{tag}"))
    except subprocess.CalledProcessError:
        pytest.skip(f"the {sanitize} sanitizer runtime is not available to g++ on this box")
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0", ASAN_OPTIONS="detect_leaks=0")
    r = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1800, env=env)
    assert r.returncode == 0, r.stdout[-3000:]
    assert "Sanitizer" not in r.stdout and "runtime error" not in r.stdout, r.stdout[-3000:]
    assert r.stdout.count("ongrid call") == 4 and "nan" not in r.stdout.lower(), r.stdout[-3000:]
