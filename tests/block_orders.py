"""Domain shapes and block orders shared by the uniform-grid table tests (tests/test_uniform_tables.py) and the device tests
on them (tests/test_gpu_block_orders.py), so that both always exercise the same cases."""
import numpy as np

import cup2d_b200

# (bpdx, bpdy, level): 6x4, 5x3, 3x1, 14x2 blocks (one tile row, partial tiles next to others along x); 10x6 and 6x10
# blocks (two tile rows and columns, tiles that stop partway in x and in y next to other tiles, tiles off every wall);
# 8x4 blocks (the rectangular shape of tests/test_gpu_parity.py, whole tiles)
SHAPES = [(3, 2, 1), (5, 3, 0), (3, 1, 0), (7, 1, 1), (5, 3, 1), (3, 5, 1), (2, 1, 2)]
ORDERS = ["hilbert", "row", "col", "random", "rhilbert"]


def make_order(bpdx, bpdy, level, kind, seed=0):
    """(i, j) of every block: the Hilbert order, row-major (i fastest), column-major (j fastest), a seeded random
    permutation, or the Hilbert order reversed (same locality, tiles met in another order)"""
    nbx, nby = bpdx << level, bpdy << level
    k = np.arange(nbx * nby)
    if kind in ("hilbert", "rhilbert"):
        o = cup2d_b200.block_order(bpdx, bpdy, level)
        o = o[::-1] if kind == "rhilbert" else o
    elif kind == "row":
        o = np.stack([k % nbx, k // nbx], axis=1)
    elif kind == "col":
        o = np.stack([k // nby, k % nby], axis=1)
    elif kind == "random":
        rng = np.random.default_rng(1000 * nbx + nby + seed)
        o = np.stack([k % nbx, k // nbx], axis=1)[rng.permutation(len(k))]
    else:
        raise ValueError(kind)
    return np.ascontiguousarray(o, dtype=np.int32)
