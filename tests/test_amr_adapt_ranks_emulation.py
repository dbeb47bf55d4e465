"""adapt() and regrid on distributed multi-level contexts (tests/amr_adapt_ranks.py), on the CPU against a g++ build of the
product sources (tests/host_emu/build.py build_full) with 1 to 5 ranks running as threads of one process: their device
buffers are mapped into each other through the emulated IPC handles, so the tag gather, the peer barriers and the transfer's
reads of other ranks' old blocks run as they do across GPUs.  Against a plain context: the new list, the new partition
(the reference's rule, restated in amr_adapt_ranks.rule), the fields bit for bit and two steps afterwards."""
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


def _run(code, lib, **env):
    r = subprocess.run([sys.executable, "-c", "import sys\nsys.path.insert(0, %r)\n" % HERE + code], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=1800, env=dict(os.environ, CUP2D_B200_LIB=lib, **env), cwd=ROOT)
    assert r.returncode == 0 and "DONE" in r.stdout, r.stdout[-3000:]
    return r.stdout


# per case: the partitions run and the properties they must show between them
#   split_children  a refined parent whose children land on two new ranks
#   third_rank_lab  a refined parent whose lab rows read blocks of a rank that neither owns it nor computes its children
#   group_base_left / _right  a compressed group split across a rank boundary, its base sibling left / right of it
#   producer_empty  a rank all of whose old blocks are non-base siblings of groups based elsewhere (min n == 0)
#   full / flux_both  the full-rebalance branch; the flux branch with flux in both directions
PLAN = {
    "runsh": (("1", "5even"), ("split_children", "third_rank_lab", "full")),
    "runsh_device_tags": (("3even",), ("full",)),
    "three_level": (("4uneven", "base_left", "base_right", "empty"),
                    ("split_children", "third_rank_lab", "group_base_left", "group_base_right", "producer_empty", "full")),
    "generated": (("2even",), ("split_children", "full")),
    "flux": (("3flux",), ("flux_both",)),
}


@pytest.mark.parametrize("name", list(PLAN))
def test_distributed_adapt_equals_the_plain_context_emulated(emulated_library, name):
    labels, wanted = PLAN[name]
    code = r'''
import amr_adapt_ranks as ar
c = ar.case(%r)
one = ar.one_rank(c)
parts = ar.partitions(c, one["blocks"])
seen, worst = set(), 0.0
for label in %r:
    rb = parts[label]
    res = ar.on_threads(len(rb) - 1, lambda r, d, b: ar.on_rank(c, r, rb, d, barrier=b))
    worst = max(worst, ar.compare(c, one, res, rb))
    prop = ar.properties(c["blocks"], one["blocks"], rb, res[0]["rb"], c["bpdx"], c["bpdy"])
    seen |= {k for k, v in prop.items() if v}
    print(label, rb.tolist(), "->", res[0]["rb"].tolist(), sorted(seen), flush=True)
assert set(%r) <= seen, seen
print("WORST", worst, "DONE")
''' % (name, labels, wanted)
    print(_run(code, emulated_library)[-600:])


def test_distributed_regrid_and_repartition_of_an_unchanged_mesh_emulated(emulated_library):
    """regrid onto the adapted list on three ranks; an unchanged mesh whose partition the rule changes (changed = 1, every
    block copied to its new rank); an unchanged mesh and partition (changed = 0, every field untouched, tmpV included)"""
    code = r'''
import numpy as np
import amr_adapt_ranks as ar
from cup2d_b200.amr import adapt_mesh
c = ar.case("three_level")
new = adapt_mesh(c["blocks"], c["bpdx"], c["bpdy"], c["level_max"], c["linf"], c["rtol"], c["ctol"])
one = ar.one_rank(c, regrid_to=new)
rb = ar.partitions(c, new)["3even"]
ar.compare(c, one, ar.on_threads(3, lambda r, d, b: ar.on_rank(c, r, rb, d, barrier=b, regrid_to=new)), rb)
# unchanged mesh: no tag refines or compresses
c = dict(c, linf=np.full(len(c["blocks"]), 0.5))
nb = len(c["blocks"])
one = ar.one_rank(c, steps=1)
assert not one["changed"] and np.array_equal(one["blocks"], c["blocks"])
skew = np.array([0, 10, nb], dtype=np.int64)        # 10 / 177 blocks: max / min > 1.01, rebalanced to 94 / 93
res = ar.on_threads(2, lambda r, d, b: ar.on_rank(c, r, skew, d, barrier=b, steps=1))
ar.compare(c, one, res, skew)
assert all(p["changed"] for p in res) and res[0]["rb"].tolist() == [0, 94, nb]
fixed = ar.rule(ar.produced(c["blocks"], c["blocks"], np.array([0, 94, nb])))
assert fixed.tolist() == [0, 94, nb]
def noop(rank, dist, barrier):
    from cup2d_b200.amr import AmrSimulation
    s = AmrSimulation.distributed(c["blocks"], 1, 1, c["h0"], ar.NU, rank, fixed, dist)
    b0, b1 = int(fixed[rank]), int(fixed[rank + 1])
    for n, a in c["fields"].items():
        s.upload(n, a[b0:b1])
    changed = s.adapt(c["rtol"], c["ctol"], c["level_max"], block_linf=c["linf"][b0:b1], dist=dist)
    same = all(np.array_equal(s.download(n), c["fields"][n][b0:b1]) for n in ar.FIELDS)
    s.step(cfl=0.5, max_iter=3)      # the peers are the old ones, still attached
    barrier(); s.close()
    return changed, same
assert ar.on_threads(2, noop) == [(False, True), (False, True)]
print("DONE")
'''
    _run(code, emulated_library)


def test_distributed_adapt_errors_emulated(emulated_library):
    """ranks that pass different level_max: CUP2D_ECOMM on both within the 300 ms wait bound, contexts still usable; calls
    between an adapt that moved the fields and the re-attach: CUP2D_ESTATE, no fault; fewer new blocks than ranks:
    CUP2D_EINVAL on every rank, contexts untouched"""
    code = r'''
import ctypes as C, time
import numpy as np
import amr_adapt_ranks as ar
from cup2d_b200.lib import Cup2dError
c = ar.case("three_level")
nb = len(c["blocks"]); rb = np.array([0, nb // 2, nb], dtype=np.int64)
def run(rank, dist, barrier):
    from cup2d_b200.amr import AmrSimulation
    s = AmrSimulation.distributed(c["blocks"], 1, 1, c["h0"], ar.NU, rank, rb, dist)
    b0, b1 = int(rb[rank]), int(rb[rank + 1])
    for n, a in c["fields"].items():
        s.upload(n, a[b0:b1])
    linf = c["linf"][b0:b1]
    t0 = time.time()
    rc = s.lib.cup2d_amr_adapt(s._h, linf.ctypes.data_as(C.POINTER(C.c_double)), c["rtol"], c["ctol"], c["level_max"] + rank, None, None)
    msg = s.lib.cup2d_last_error().decode()
    dt = time.time() - t0
    kept = all(np.array_equal(s.download(n), c["fields"][n][b0:b1]) for n in ar.FIELDS)
    changed = C.c_int32()
    rc2 = s.lib.cup2d_amr_adapt(s._h, linf.ctypes.data_as(C.POINTER(C.c_double)), c["rtol"], c["ctol"], c["level_max"], None, C.byref(changed))
    codes = []
    for call in (lambda: s.step(cfl=0.5, max_iter=3), lambda: s.compute_dt(0.5), lambda: s.poisson_solve(max_iter=3),
                 lambda: s.forces([])):
        try:
            call()
            codes.append(0)
        except Cup2dError as e:
            codes.append(str(e).split(":")[0])
    s._after_regrid(bool(changed.value), dist)     # the re-attach; then steps run
    s.step(cfl=0.5, max_iter=3)
    barrier(); s.close()
    return rc, msg, dt, kept, rc2, changed.value, codes
res = ar.on_threads(2, run)
print(res)
for rc, msg, dt, kept, rc2, changed, codes in res:
    assert rc == -5 and "different arguments" in msg and dt < 60 and kept
    assert rc2 == 0 and changed == 1
    assert codes[:3] == ["cup2d error -4"] * 3, codes
# fewer new blocks than ranks: four level-1 blocks compress into one
b4 = ar.case("three_level")
b4 = dict(b4, blocks=np.array([(1, 0, 0), (1, 1, 0), (1, 1, 1), (1, 0, 1)], dtype=np.int32), level_max=3, linf=np.zeros(4),
          fields=ar.seeded_fields(4, 1))
rb4 = np.array([0, 2, 4], dtype=np.int64)
def few(rank, dist, barrier):
    from cup2d_b200.amr import AmrSimulation
    s = AmrSimulation.distributed(b4["blocks"], 1, 1, 1 / 8, ar.NU, rank, rb4, dist)
    for n, a in b4["fields"].items():
        s.upload(n, a[2 * rank:2 * rank + 2])
    try:
        s.adapt(0.5, 0.1, 3, block_linf=np.zeros(2), dist=dist)
        err = "no error"
    except Cup2dError as e:
        err = str(e)
    kept = all(np.array_equal(s.download(n), b4["fields"][n][2 * rank:2 * rank + 2]) for n in ar.FIELDS)
    kept &= np.array_equal(s.block_list(), b4["blocks"]) and s.rank_begin().tolist() == [0, 2, 4]
    s.step(cfl=0.5, max_iter=3)
    barrier(); s.close()
    return err, kept
res = ar.on_threads(2, few)
print(res)
assert all("error -1" in e and "fewer blocks than ranks" in e and k for e, k in res), res
print("DONE")
'''
    _run(code, emulated_library, CUP2D_COMM_TIMEOUT_MS="300")
