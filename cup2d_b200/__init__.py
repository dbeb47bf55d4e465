"""cup2d_b200 — H100-native (sm_90a) implementation of CUP2D's per-timestep hot path.

The product is the C-ABI shared library libcup2d_b200.so (include/cup2d_b200.h, sources in
cup2d_b200/csrc/).  This package is the thin host-side mirror used by tests and bench.py: ctypes
bindings (`lib`) and `Simulation`, which follows the reference driver's configuration names
(bpdx, bpdy, levelStart, extent, nu, CFL, ... main.cpp:6321-6337).  There is no CPU fallback:
importing works anywhere, creating a Simulation without an sm_90 GPU raises.
"""
from .lib import Cup2dError, load_library, FIELDS  # noqa: F401
from .sim import Simulation, block_order, to_blocks, from_blocks  # noqa: F401
