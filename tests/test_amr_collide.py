"""CPU tests of the collision model on multi-level meshes: the oracle (tests/amr_collision_oracle.py) against the reference's own
collision model on its run.sh mesh (tests/golden/amrcollide_lmax8.npz), and the device code (tests/test_gpu_amr_collide.py) on
the emulated library."""
import os
import subprocess
import sys

import numpy as np
import pytest

import amr_collision_oracle as co

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def calls(golden_dir):
    sys.path.insert(0, golden_dir)
    import make_collide_golden
    return make_collide_golden.load(os.path.join(golden_dir, "amrcollide_lmax8.npz"))


def test_oracle_equals_the_reference_bit_for_bit(calls):
    for c in calls:
        uvw, buf, _ = co.collide(c["blocks"], c["h0"], c["shapes"])
        assert np.array_equal(buf, c["sums20"]), c["config"]
        assert np.array_equal(uvw, c["uvw_after"]), c["config"]


def test_fixture_has_an_impulse_and_a_receding_pair(calls):
    """head to head: the impulse changes both fish; tail to tail: the pair passes the mass and distance tests, projVel <= 0"""
    seen = set()
    for c in calls:
        before = np.array([[s[n] for n in ("u", "v", "omega")] for s in c["shapes"]])
        b = co.branches(c["sums20"], c["shapes"])[0, 1]
        assert b == {"head": "impulse", "tail": "receding"}[c["config"]]
        assert np.array_equal(before, c["uvw_after"]) == (b == "receding")
        assert (c["sums20"][:, [3, 6, 9, 13, 16, 19]] == 0).all()
        seen.add(b)
    assert seen == {"impulse", "receding"}


def test_device_collide_on_the_emulated_library():
    """tests/test_gpu_amr_collide.py on a g++ build of the product sources (tests/host_emu/build.py build_full)"""
    sys.path.insert(0, os.path.join(HERE, "host_emu"))
    import build
    lib = build.build_full()
    env = dict(os.environ, CUP2D_B200_LIB=lib)
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(HERE, "test_gpu_amr_collide.py"), "-m", "gpu", "-q",
                        "-p", "no:cacheprovider"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env,
                       timeout=1800, cwd=ROOT)
    tail = r.stdout[-2000:]
    assert r.returncode == 0 and " passed" in tail and "failed" not in tail and "skipped" not in tail, tail


sanitizers = pytest.mark.skipif(os.environ.get("CUP2D_TEST_SANITIZERS") != "1", reason="sanitizer builds are opt-in: CUP2D_TEST_SANITIZERS=1")


@sanitizers
@pytest.mark.parametrize("sanitize", ["thread", "address,alignment,bounds"])
def test_collide_under_sanitizers(sanitize):
    """tests/host_emu/collide_driver.cpp (two overlapping ongrid bodies across a level jump, two collide calls) linked against
    the emulated product sources built with ThreadSanitizer / AddressSanitizer: no report, no NaN from never-written memory"""
    sys.path.insert(0, os.path.join(HERE, "host_emu"))
    import build
    build.build_full()
    tag = "tsan" if sanitize == "thread" else "asan"
    srcs = [os.path.join(build.FULL, f) for f in sorted(os.listdir(build.FULL)) if f.endswith(".cpp")]
    exe = os.path.join(build.FULL, f"collide_{tag}_driver")
    try:
        build._compile_link(["-O1", "-g", "-std=c++20", "-pthread", f"-fsanitize={sanitize}",
                             *([] if sanitize == "thread" else ["-fno-sanitize-recover=all"]), "-w", "-DEMU_ALL_COOP",
                             "-I", build.FULL, "-I", os.path.join(HERE, "host_emu")],
                            [os.path.join(HERE, "host_emu", "collide_driver.cpp"), *srcs], exe,
                            os.path.join(build.FULL, f"obj_collide_{tag}"))
    except subprocess.CalledProcessError:
        pytest.skip(f"the {sanitize} sanitizer runtime is not available to g++ on this box")
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0", ASAN_OPTIONS="detect_leaks=0")
    r = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1800, env=env)
    assert r.returncode == 0, r.stdout[-3000:]
    assert "Sanitizer" not in r.stdout and "runtime error" not in r.stdout, r.stdout[-3000:]
    assert r.stdout.count("collide call") == 2 and "nan" not in r.stdout.lower(), r.stdout[-3000:]
