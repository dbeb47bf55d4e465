"""The device tests on generated meshes (tests/test_gpu_amr_meshes.py) on the CPU, against the emulated build of the product
sources (tests/host_emu/build.py build_full).  A subset: one rectangular mesh in random order (operators in both kernel modes,
tagging, dump, adapt(), the step against the composed oracle and the enqueued step against the blocking one) and the
1025-block mesh, whose reductions run one block past a 1024-thread pass.  The whole file, without the mesh above 8192
blocks: tools/run_emulated_gpu_tests.sh."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

SUBSET = "(1x3_mixed and random) or n1025"


def test_generated_meshes_on_the_emulated_library():
    sys.path.insert(0, os.path.join(HERE, "host_emu"))
    import build
    lib = build.build_full()
    env = dict(os.environ, CUP2D_B200_LIB=lib)
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(HERE, "test_gpu_amr_meshes.py"), "-m", "gpu", "-q",
                        "-k", SUBSET, "-p", "no:cacheprovider"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env, timeout=1800, cwd=ROOT)
    tail = r.stdout[-3000:]
    assert r.returncode == 0, tail
    assert " passed" in tail and "failed" not in tail
    assert int(tail.split(" passed")[0].split()[-1]) == 13, tail
