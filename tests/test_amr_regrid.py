"""CPU tests of adapt() on multi-level meshes: the oracle's decision and field transfer (tests/amr_adapt_oracle.py) and the
library's host-side decision (cup2d_amr_adapt_mesh) and refinement labs (plan kinds 4 / 5) against the reference's own adapt()
on its run.sh mesh (tests/golden/amrregrid_lmax8.npz), and the device regrid on the emulated library."""
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp

import amr_adapt_oracle as ao
from cup2d_b200.amr import AmrPlan, adapt_mesh

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
FIELDS = (("vel", "vector"), ("vold", "vector"), ("pres", "scalar"), ("pold", "scalar"), ("chi", "scalar"), ("tmp", "scalar"))


@pytest.fixture(scope="module")
def g(golden_dir):
    sys.path.insert(0, golden_dir)
    import make_regrid_golden
    return make_regrid_golden.load(os.path.join(golden_dir, "amrregrid_lmax8.npz"))


def test_oracle_decision_and_order_equal_the_reference(g):
    mesh = ao.Mesh(g["blocks"], int(g["bpdx"]), int(g["bpdy"]))
    new = ao.amr_adapt_mesh(mesh, g["block_linf"], float(g["rtol"]), float(g["ctol"]), int(g["level_max"]))
    assert np.array_equal(new, g["new_blocks"])
    newset = set(map(tuple, new.tolist()))
    refined = {l for l, i, j in g["blocks"].tolist() if (l + 1, 2 * i, 2 * j) in newset}
    assert len(refined) >= 3


def test_oracle_transfer_bit_exact(g):
    mesh = ao.Mesh(g["blocks"], int(g["bpdx"]), int(g["bpdy"]))
    out = ao.amr_regrid(mesh, g["new_blocks"], {n: (g[n], k) for n, k in FIELDS})
    for n, _ in FIELDS:
        assert np.array_equal(out[n], g["new_" + n]), n


def test_adapt_mesh_equals_the_reference(g):
    new = adapt_mesh(g["blocks"], g["bpdx"], g["bpdy"], g["level_max"], g["block_linf"], g["rtol"], g["ctol"])
    assert np.array_equal(new, g["new_blocks"])


def _random_meshes():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import bench_amr
    return [(bench_amr.three_level_mesh(b, r1=r1, r2=r2, centre=c), 1, 1, b + 3)
            for b, r1, r2, c in ((3, 0.3, 0.15, (0.45, 0.55)), (3, 0.4, 0.2, (0.1, 0.9)), (4, 0.25, 0.1, (0.7, 0.3)))]


def test_adapt_mesh_equals_the_oracle_on_random_tags(g):
    """the golden mesh and three synthetic three-level meshes, a few hundred seeded tag vectors: the library's decision equals
    the oracle's (blocks and order), and the result is a valid 2:1-balanced mesh (cup2d_amr_plan_create accepts it)"""
    rng = np.random.default_rng(7)
    cases = [(g["blocks"], int(g["bpdx"]), int(g["bpdy"]), int(g["level_max"]))] + _random_meshes()
    changed = compressed = 0
    for blocks, bx, by, lmax in cases:
        mesh = ao.Mesh(blocks, bx, by)
        for _ in range(80):
            linf = rng.uniform(0, 1, len(blocks)) * rng.choice([1.0, 0.0], len(blocks), p=[0.9, 0.1])
            rtol, ctol = sorted(rng.uniform(0, 1, 2))[::-1]
            want = ao.amr_adapt_mesh(mesh, linf, rtol, ctol, lmax)
            got = adapt_mesh(blocks, bx, by, lmax, linf, rtol, ctol)
            assert np.array_equal(got, want)
            AmrPlan(got, bx, by).close()
            changed += not np.array_equal(got, blocks)
            compressed += any((l + 1, 2 * i, 2 * j) in mesh.index for l, i, j in got.tolist())
    assert changed > 200 and compressed > 20


def test_adapt_mesh_rejects_bad_input():
    from cup2d_b200 import lib as L
    lib = L.load_library()
    import ctypes as C
    b = np.array([[0, 0, 0], [0, 0, 0]], dtype=np.int32)
    linf = np.zeros(2)
    n = lib.cup2d_amr_adapt_mesh(2, b.ctypes.data_as(C.POINTER(C.c_int32)), 2, 1, 3, linf.ctypes.data_as(C.POINTER(C.c_double)),
                                 1.0, 0.5, None)
    assert n == -1 and b"duplicated" in lib.cup2d_last_error()


@pytest.mark.parametrize("which,name,field,kind", [(4, "lab_vel", "vel", "vector"), (5, "lab_pres", "pres", "scalar")])
def test_refinement_lab_tables_reproduce_reference_labs(g, which, name, field, kind):
    """kinds 4 / 5 (the {-1,-1,2,2,tensorial} labs adapt() refines from) applied to the golden fields: the reference's labs to
    1e-13, and empty rows exactly where the oracle's lab is unwritten (here: nowhere, corners included)"""
    plan = AmrPlan(g["blocks"], int(g["bpdx"]), int(g["bpdy"]))
    rowptr, sb, sc, w = plan.stencil(which)
    plan.close()
    nb, dim = len(g["blocks"]), 2 if which == 4 else 1
    T = sp.csr_matrix((w, sb.astype(np.int64) * 64 * dim + sc, rowptr), shape=(nb * 100 * dim, nb * 64 * dim))
    lab = (T @ g[field].reshape(-1)).reshape(nb, 10, 10, dim)
    empty = (np.diff(rowptr) == 0).reshape(nb, 10, 10, dim)
    olab = ao.Lab(ao.Mesh(g["blocks"], int(g["bpdx"]), int(g["bpdy"])), g[field], (-1, -1, 2, 2, True), kind)
    unwritten = np.array([np.isnan(olab.load(k)) for k in range(0, nb, 7)])
    assert np.array_equal(empty[::7], unwritten)
    want, sel = g[name], g["lab_blocks"]   # the reference's labs of the refined blocks
    assert len(sel) > 0 and not empty[sel].any()
    assert np.abs(lab[sel] - want).max() < 1e-13 * np.abs(want).max()


def test_device_regrid_on_the_emulated_library():
    """tests/test_gpu_amr_regrid.py on a g++ build of the product sources (tests/host_emu/build.py build_full)"""
    sys.path.insert(0, os.path.join(HERE, "host_emu"))
    import build
    lib = build.build_full()
    env = dict(os.environ, CUP2D_B200_LIB=lib)
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(HERE, "test_gpu_amr_regrid.py"), "-m", "gpu", "-q",
                        "-p", "no:cacheprovider"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env,
                       timeout=1800, cwd=ROOT)
    tail = r.stdout[-2000:]
    assert r.returncode == 0 and " passed" in tail and "failed" not in tail and "skipped" not in tail, tail


sanitizers = pytest.mark.skipif(os.environ.get("CUP2D_TEST_SANITIZERS") != "1", reason="sanitizer builds are opt-in: CUP2D_TEST_SANITIZERS=1")


@sanitizers
@pytest.mark.parametrize("sanitize", ["thread", "address,alignment,bounds"])
def test_regrid_under_sanitizers(sanitize):
    """tests/host_emu/regrid_driver.cpp (step, regrid with a refine and a compress, steps on the new mesh) linked against the
    emulated product sources built with ThreadSanitizer / AddressSanitizer: no report, no NaN from never-written memory"""
    sys.path.insert(0, os.path.join(HERE, "host_emu"))
    import build
    build.build_full()
    tag = "tsan" if sanitize == "thread" else "asan"
    srcs = [os.path.join(build.FULL, f) for f in sorted(os.listdir(build.FULL)) if f.endswith(".cpp")]
    exe = os.path.join(build.FULL, f"regrid_{tag}_driver")
    try:
        build._compile_link(["-O1", "-g", "-std=c++20", "-pthread", f"-fsanitize={sanitize}",
                             *([] if sanitize == "thread" else ["-fno-sanitize-recover=all"]), "-w", "-DEMU_ALL_COOP",
                             "-I", build.FULL, "-I", os.path.join(HERE, "host_emu")],
                            [os.path.join(HERE, "host_emu", "regrid_driver.cpp"), *srcs], exe,
                            os.path.join(build.FULL, f"obj_regrid_{tag}"))
    except subprocess.CalledProcessError:
        pytest.skip(f"the {sanitize} sanitizer runtime is not available to g++ on this box")
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0", ASAN_OPTIONS="detect_leaks=0")
    r = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1800, env=env)
    assert r.returncode == 0, r.stdout[-3000:]
    assert "Sanitizer" not in r.stdout and "runtime error" not in r.stdout, r.stdout[-3000:]
    assert r.stdout.count("regrid step") == 2 and "nan" not in r.stdout.lower(), r.stdout[-3000:]
