"""The body calls on distributed multi-level contexts (cup2d_amr_ongrid, _surface, _forces, _collide on
cup2d_amr_create_ranks contexts), on the CPU against a g++ build of the product sources (tests/host_emu/build.py build_full)
with the ranks running as threads of one process: their device buffers are mapped into each other through the emulated IPC
handles, so the halo pulls and the peer all-reduce run as they do across GPUs.  1, 2, 3 and 4 ranks on the reference's
run.sh records (tests/golden/amrongrid_lmax8.npz, amrforces_lmax8.npz, amrcollide_lmax8.npz) and on a synthetic
three-level mesh, against a one-rank cup2d_amr_create context and against the numbers the oracles pin
(tests/amr_bodies_ranks.py lists what is bitwise and what agrees to rounding)."""
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

sys.path.insert(0, HERE)
import amr_bodies_ranks  # noqa: E402


@pytest.fixture(scope="module")
def emulated_library():
    sys.path.insert(0, os.path.join(HERE, "host_emu"))
    import build
    return build.build_full()


def _run(code, lib, **env):
    r = subprocess.run([sys.executable, "-c", code], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600,
                       env=dict(os.environ, CUP2D_B200_LIB=lib, **env), cwd=ROOT)
    assert r.returncode == 0 and "DONE" in r.stdout, r.stdout[-3000:]
    return r.stdout


@pytest.mark.parametrize("case", amr_bodies_ranks.CASES)
def test_distributed_body_calls_equal_one_rank_emulated(emulated_library, case):
    """every partition of amr_bodies_ranks.partitions: a cut through the obstacle blocks whose chi and force labs read
    remote blocks across a level jump, a rank without obstacle blocks, a shape entirely on one rank and (two shapes sharing
    blocks) their common blocks on several ranks"""
    code = r'''
import sys
sys.path.insert(0, %r)
import amr_bodies_ranks as ar
inp = ar.case_inputs(%r)
one = ar.one_rank(inp)
parts = ar.partitions(inp, one)
prop = ar.properties(inp, one, parts)
assert sorted(parts) == [1, 2, 3, 4] and prop["empty_rank"] and prop["whole_shape"] and prop["remote_level_jump"], prop
assert prop["split_common"] or inp["kind"] != "collide", prop
worst = 0.0
for W, rb in parts.items():
    res = ar.on_threads(W, lambda r, d, b: ar.on_rank(inp, r, rb, d, barrier=b))
    worst = max(worst, ar.compare(one, res, rb))
    ar.check_pinned(inp, ar.assemble(res))
print("WORST", worst, prop, "DONE")
''' % (HERE, case)
    out = _run(code, emulated_library)
    print(out[-400:])


def test_ranks_that_pass_different_shape_counts_fail_instead_of_hanging(emulated_library):
    """two ranks call ongrid with one and with two bodies: the all-reduce compares the value counts before it adds anything,
    so both calls return CUP2D_ECOMM (and no wait runs into the CUP2D_COMM_TIMEOUT_MS bound); the same for collide"""
    code = r'''
import sys, time
sys.path.insert(0, %r)
import amr_bodies_ranks as ar
from cup2d_b200.lib import Cup2dError
inp = ar.case_inputs("runsh_ongrid")
nb = len(inp["blocks"]); rb = [0, nb // 2, nb]
def run(rank, dist, barrier):
    from cup2d_b200.amr import AmrSimulation
    sim = AmrSimulation.distributed(inp["blocks"], inp["bpdx"], inp["bpdy"], inp["h0"], inp["nu"], rank, rb, dist)
    msgs, t0 = [], time.time()
    for call in (lambda: sim.ongrid(inp["bodies"][:1 + rank]),
                 lambda: sim.collide(ar._motions_from(out10[:1 + rank]))):
        try:
            call()
            msgs.append("no error")
        except Cup2dError as e:
            msgs.append(str(e))
        if len(msgs) == 1:   # both ranks place both bodies, then disagree on the collide call
            out10 = sim.ongrid(inp["bodies"])
    barrier(); sim.close()
    return msgs, time.time() - t0
res = ar.on_threads(2, run)
print("MSG", res)
for msgs, dt in res:
    assert all("error -5" in m and "different numbers of values" in m for m in msgs), msgs
    assert dt < 60
print("DONE")
''' % (HERE,)
    _run(code, emulated_library, CUP2D_COMM_TIMEOUT_MS="300")
