#!/bin/bash
# All GPU parity tests (including the opt-in multi-level ones) on the CPU, against the g++ build of the product sources
# (tests/host_emu/; see tests/test_full_emulation.py for what this does and does not check).  About 5 minutes.
set -e
cd "$(dirname "$0")/.."
LIB=$(python -c "import sys; sys.path.insert(0, 'tests/host_emu'); import build; print(build.build_full())")
CUP2D_B200_LIB=$LIB python -m pytest tests/test_gpu_parity.py tests/test_gpu_amr.py tests/test_gpu_amr_regrid.py tests/test_gpu_amr_ongrid.py tests/test_gpu_amr_collide.py tests/test_gpu_amr_forces.py tests/test_gpu_block_orders.py tests/test_gpu_krylov_branches.py -m gpu -q \
  -k "not 1024 and not tolerance_driven and not large_grid and not reference_driver and not reference_amr and not two_ranks and not multi_chunk" "$@"
# the generated meshes (tests/amr_meshes.py), without the 9 602-block mesh, whose steps take too long emulated
CUP2D_B200_LIB=$LIB python -m pytest tests/test_gpu_amr_meshes.py -m gpu -q -k "not large" "$@"
# the sanitizer builds of the same sources (ThreadSanitizer race hunt, AddressSanitizer bounds/alignment hunt)
CUP2D_TEST_SANITIZERS=1 python -m pytest tests/test_full_emulation.py -q -k "sanitizer"
