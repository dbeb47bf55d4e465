#!/bin/bash
# A/B builds of the advect kernel (run here, before gpurun; the .so files travel with the snapshot):
#   cup2d_b200/libcup2d_b200_<tag>.so = the product library with advect.cu (and amr_fast.cu) compiled with extra defines.
# Select at run time with CUP2D_B200_LIB=<path> (cup2d_b200/lib.py).
set -e
cd "$(dirname "$0")/../cup2d_b200/csrc"
make > /dev/null
OBJ=$(make -s --eval 'objs: ; @echo $(OBJ)' objs) # the objects the Makefile links into the product library
NV="nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -Xcompiler -fPIC -Xptxas -v --expt-extended-lambda -ccbin /usr/bin/g++"
build() { # tag, defines
  $NV $2 -c advect.cu -o advect_v_$1.o 2> advect_$1.ptxas.log
  nvcc -gencode arch=compute_90a,code=sm_90a -shared -o ../libcup2d_b200_$1.so ${OBJ/advect.o/advect_v_$1.o} -ccbin /usr/bin/g++
  echo "$1: $(grep -c 'bytes spill' advect_$1.ptxas.log) kernels, max regs $(grep -o 'Used [0-9]* registers' advect_$1.ptxas.log | sort -k2 -n | tail -1)"
  rm -f advect_v_$1.o
}
build tma "-DCUP2D_ADV_LDGSTS=0"
# the row-mapped stencil kernels with per-lane edge-row loads and all ghost cells from global memory (rows.cuh, round-1 form)
$NV -DCUP2D_ROWS_COOP=0 -c poisson.cu -o poisson_v_nocoop.o 2> poisson_nocoop.ptxas.log
$NV -DCUP2D_ROWS_COOP=0 -c pressure.cu -o pressure_v_nocoop.o 2> pressure_nocoop.ptxas.log
NOCOOP=${OBJ/poisson.o/poisson_v_nocoop.o}
NOCOOP=${NOCOOP/pressure.o/pressure_v_nocoop.o}
nvcc -gencode arch=compute_90a,code=sm_90a -shared -o ../libcup2d_b200_nocoop.so $NOCOOP -ccbin /usr/bin/g++
rm -f poisson_v_nocoop.o pressure_v_nocoop.o
