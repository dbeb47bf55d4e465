"""CPU tests of adapt()'s tagging on the fused kernel: tests/test_gpu_amr_tags_fast.py on a g++ build of the product sources
(tests/host_emu/build.py build_full), whose kernels run thread by thread on the host; distributed contexts of 2 and 3 ranks
(threads of one process) with cuts on level interfaces against the plain context, bit for bit; and
tests/host_emu/tags_driver.cpp, which checks that tagging and adapt on fast and distributed contexts allocate none of the
full per-cell tables (under CUP2D_TEST_SANITIZERS=1 also with ThreadSanitizer and AddressSanitizer)."""
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def emulated_library():
    sys.path.insert(0, os.path.join(HERE, "host_emu"))
    import build
    return build.build_full()


def test_fast_tagging_on_the_emulated_library(emulated_library):
    env = dict(os.environ, CUP2D_B200_LIB=emulated_library)
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(HERE, "test_gpu_amr_tags_fast.py"), "-m", "gpu", "-q",
                        "-p", "no:cacheprovider"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env,
                       timeout=3000, cwd=ROOT)
    tail = r.stdout[-3000:]
    assert r.returncode == 0 and " passed" in tail and "failed" not in tail and "skipped" not in tail, tail


@pytest.mark.parametrize("nranks", [2, 3])
def test_distributed_tagging_with_cuts_on_level_interfaces(emulated_library, nranks):
    code = r'''
import numpy as np
import amr_adapt_ranks as ar
import amr_meshes as M
import bench_amr
from cup2d_b200.amr import AmrSimulation, AmrPlan
b = M.reference_order(bench_amr.three_level_mesh(3, r1=0.3, r2=0.15, centre=(0.45, 0.55)), 1, 1, 6).astype(np.int32)
nb, W = len(b), %d
f = ar.seeded_fields(nb, 21)
f["chi"] = np.where(f["chi"] > 0.98, f["chi"], 0.0)
rtol, lmax = 40.0, 6
# cuts between a block and the next one in the list that lie across a level interface: the two blocks are neighbours of
# different levels, so each rank's labs read the other's blocks through coarse-fine ghost rows
n8 = AmrPlan(b, 1, 1).neighbours()
cand = [k for k in range(1, nb) if b[k, 0] != b[k - 1, 0] and (n8[k] == -2).any() | (n8[k] == -3).any()]
assert len(cand) >= W - 1, cand
cuts = [cand[(len(cand) * (r + 1)) // W] for r in range(W - 1)]
rb = np.array([0] + sorted(set(cuts)) + [nb], dtype=np.int64)
assert len(rb) == W + 1
plain = AmrSimulation(b, 1, 1, 1 / 8, ar.NU)
plain.upload("vel", f["vel"]); plain.upload("chi", f["chi"])
want, want_tmp = plain.adapt_tags(rtol, lmax), plain.download("tmp")
plain.close()
assert (want == 2 * rtol).any()
def run(rank, dist, barrier):
    s = AmrSimulation.distributed(b, 1, 1, 1 / 8, ar.NU, rank, rb, dist)
    b0, b1 = int(rb[rank]), int(rb[rank + 1])
    s.upload("vel", f["vel"][b0:b1]); s.upload("chi", f["chi"][b0:b1])
    out = (s.adapt_tags(rtol, lmax), s.download("tmp"))
    barrier(); s.close()
    return out
res = ar.on_threads(W, run)
bits = lambda a: np.ascontiguousarray(a).view(np.uint64)
assert np.array_equal(bits(np.concatenate([r[0] for r in res])), bits(want))
assert np.array_equal(bits(np.concatenate([r[1] for r in res])), bits(want_tmp))
print(rb.tolist(), "DONE")
''' % nranks
    r = subprocess.run([sys.executable, "-c", "import sys\nsys.path.insert(0, %r)\n" % HERE + code], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=1800, env=dict(os.environ, CUP2D_B200_LIB=emulated_library), cwd=ROOT)
    assert r.returncode == 0 and "DONE" in r.stdout, r.stdout[-3000:]


def _driver(sanitize):
    sys.path.insert(0, os.path.join(HERE, "host_emu"))
    import build
    build.build_full()
    tag = {None: "plain", "thread": "tsan"}.get(sanitize, "asan")
    srcs = [os.path.join(build.FULL, f) for f in sorted(os.listdir(build.FULL)) if f.endswith(".cpp")]
    exe = os.path.join(build.FULL, f"tags_{tag}_driver")
    flags = ["-O1", "-g", "-std=c++20", "-pthread", "-w", "-I", build.FULL, "-I", os.path.join(HERE, "host_emu")]
    if sanitize:
        flags += [f"-fsanitize={sanitize}", "-DEMU_ALL_COOP"] + ([] if sanitize == "thread" else ["-fno-sanitize-recover=all"])
    build._compile_link(flags, [os.path.join(HERE, "host_emu", "tags_driver.cpp"), *srcs], exe,
                        os.path.join(build.FULL, f"obj_tags_{tag}"))
    return exe


def _run_driver(exe):
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0", ASAN_OPTIONS="detect_leaks=0")
    r = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1800, env=env)
    assert r.returncode == 0, r.stdout[-3000:]
    assert "Sanitizer" not in r.stdout and "runtime error" not in r.stdout, r.stdout[-3000:]
    assert r.stdout.count("no full tables") == 2 and "nan" not in r.stdout.lower(), r.stdout[-3000:]


def test_no_full_tables_on_fast_and_distributed_contexts():
    _run_driver(_driver(None))


@pytest.mark.skipif(os.environ.get("CUP2D_TEST_SANITIZERS") != "1", reason="sanitizer builds are opt-in: CUP2D_TEST_SANITIZERS=1")
@pytest.mark.parametrize("sanitize", ["thread", "address,alignment,bounds"])
def test_tags_driver_under_sanitizers(sanitize):
    try:
        exe = _driver(sanitize)
    except subprocess.CalledProcessError:
        pytest.skip(f"the {sanitize} sanitizer runtime is not available to g++ on this box")
    _run_driver(exe)
