"""CPU test of adapt() in one call (cup2d_amr_adapt): tests/test_gpu_amr_adapt.py on a g++ build of the product sources
(tests/host_emu/build.py build_full), whose kernels run thread by thread on the host."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def test_device_adapt_on_the_emulated_library():
    sys.path.insert(0, os.path.join(HERE, "host_emu"))
    import build
    lib = build.build_full()
    env = dict(os.environ, CUP2D_B200_LIB=lib)
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(HERE, "test_gpu_amr_adapt.py"), "-m", "gpu", "-q",
                        "-p", "no:cacheprovider"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env,
                       timeout=1800, cwd=ROOT)
    tail = r.stdout[-3000:]
    assert r.returncode == 0 and " passed" in tail and "failed" not in tail and "skipped" not in tail, tail
