"""The enqueued multi-level steps (cup2d_amr_step_enqueue and its companions) on the CPU: tests/test_gpu_amr_step_graph.py
run against the emulated build of the product sources (tests/host_emu/build.py build_full), where every enqueue takes the
direct path — dt rule, pressure means and Krylov stopping on the device, no graphs.  The graph tests of that file need a GPU
and are left out here, and so is part of the rest: each emulated step takes tens of seconds, so the run.sh mesh and the
synthetic mesh share out the remaining checks."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


SUBSET = ("(enqueued_steps_match and runsh) or (pressure_enqueue and synthetic) or (six_enqueues and synthetic and True) "
          "or (regrid_between and True) or error_codes")


def test_enqueued_steps_on_the_emulated_library():
    sys.path.insert(0, os.path.join(HERE, "host_emu"))
    import build
    lib = build.build_full()
    env = dict(os.environ, CUP2D_B200_LIB=lib)
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(HERE, "test_gpu_amr_step_graph.py"), "-m", "gpu", "-q",
                        "-k", SUBSET, "-p", "no:cacheprovider"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env, timeout=1800, cwd=ROOT)
    tail = r.stdout[-3000:]
    assert r.returncode == 0, tail
    assert " passed" in tail and "failed" not in tail
    assert int(tail.split(" passed")[0].split()[-1]) == 7, tail
