"""Device tests of the body calls on distributed multi-level contexts (cup2d_amr_ongrid, _surface, _forces and _collide on
cup2d_amr_create_ranks contexts).  On one GPU a one-rank distributed context runs the slot-numbered tables and the
halo-aware labs and must give the plain context's results bit for bit (its all-reduce is a no-op, so the vector all-reduce
kernel itself runs only with two or more ranks: on two or more GPUs below, and on the CPU in
tests/test_amr_bodies_ranks_emulation.py).  The comparisons are those of tests/amr_bodies_ranks.py."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import amr_bodies_ranks as ar

pytestmark = [pytest.mark.gpu]
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.mark.parametrize("case", ar.CASES)
def test_one_rank_distributed_context_equals_the_plain_context(case):
    inp = ar.case_inputs(case)
    one = ar.one_rank(inp)
    rb = np.array([0, len(inp["blocks"])], dtype=np.int64)
    res = ar.on_rank(inp, 0, rb, None)
    assert ar.compare(one, [res], rb) == 0.0
    ar.check_pinned(inp, res)


def test_ranks_on_several_gpus():
    """the comparison of the emulation test on real GPUs, one process per GPU (skipped on a one-GPU box)"""
    import torch
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs 2 GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(min(n, 4)),
                        "--master-addr", "127.0.0.1", "--master-port", "29579", os.path.join(HERE, "amr_bodies_ranks.py")],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900, env=dict(os.environ))
    assert r.returncode == 0 and "BODIES_RANKS_OK" in r.stdout, r.stdout[-3000:]


def test_replicated_contexts_still_refuse_the_body_calls():
    """contexts of cup2d_amr_set_ranks (the operators replicated on every rank) keep CUP2D_ESTATE for all four calls"""
    from cup2d_b200 import lib as L
    inp = ar.case_inputs("runsh_collide0")
    from cup2d_b200.amr import AmrSimulation
    sim = AmrSimulation(inp["blocks"], inp["bpdx"], inp["bpdy"], inp["h0"], inp["nu"])
    for k, s in enumerate(inp["shapes"]):
        sim.shape_set(k, s["ids"], s["chi"], s["udef"])
        sim.shape_set_dist(k, s["dist"])
    nb = len(inp["blocks"])
    rb = np.array([0, nb // 2, nb], dtype=np.int64)
    L.check(sim.lib.cup2d_amr_set_ranks(sim._h, 0, 2, rb.ctypes.data_as(C.POINTER(C.c_int64))))
    out = np.zeros(64 * 23)
    P = C.POINTER(C.c_double)
    assert sim.lib.cup2d_amr_ongrid(sim._h, 1, (L.Body * 1)(), out.ctypes.data_as(P)) == -4
    assert sim.lib.cup2d_amr_surface(sim._h, 2) == -4
    assert sim.lib.cup2d_amr_forces(sim._h, 2, (L.Rigid * 2)(), out.ctypes.data_as(P)) == -4
    assert sim.lib.cup2d_amr_collide(sim._h, 2, (L.Rigid * 2)(), out.ctypes.data_as(P)) == -4
    assert not out.any()
    sim.close()
