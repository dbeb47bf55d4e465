"""GPU tests of adapt() and regrid on distributed multi-level contexts (cup2d_amr_adapt / cup2d_amr_regrid on
cup2d_amr_create_ranks contexts; tests/amr_adapt_ranks.py): on one H100 a one-rank distributed context adapts and regrids
bit for bit like the plain context and then steps bit for bit like it, which runs the peer-addressed transfer kernels on the
hardware with rank 0 reading itself; on two to four GPUs the same comparison with one process per GPU."""
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import amr_adapt_ranks as ar  # noqa: E402

pytestmark = [pytest.mark.gpu]


@pytest.mark.parametrize("name", ar.CASES)
def test_one_rank_distributed_adapt_equals_the_plain_context(name):
    c = ar.case(name)
    one = ar.one_rank(c)
    rb = np.array([0, len(c["blocks"])], dtype=np.int64)
    got = ar.on_rank(c, 0, rb, None)
    ar.compare(c, one, [got], rb)
    assert got["changed"] == one["changed"]


@pytest.mark.parametrize("name", ("runsh", "three_level"))
def test_one_rank_distributed_regrid_equals_the_plain_context(name):
    from cup2d_b200.amr import adapt_mesh
    c = ar.case(name)
    new = adapt_mesh(c["blocks"], c["bpdx"], c["bpdy"], c["level_max"], c["linf"], c["rtol"], c["ctol"])
    one = ar.one_rank(c, regrid_to=new)
    rb = np.array([0, len(c["blocks"])], dtype=np.int64)
    ar.compare(c, one, [ar.on_rank(c, 0, rb, None, regrid_to=new)], rb)


def test_ranks_on_several_gpus():
    import torch
    n = min(torch.cuda.device_count(), 4)
    if n < 2:
        pytest.skip("needs at least two GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--standalone", f"--nproc-per-node={n}",
                        os.path.join(HERE, "amr_adapt_ranks.py")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True, timeout=1800, cwd=ROOT)
    assert r.returncode == 0 and "ADAPT_RANKS_OK" in r.stdout, r.stdout[-3000:]
