# TEST INFRASTRUCTURE — the device form of the reference's multi-level fish loop and the step recorder it is checked with.
#
#   make -f amrdevice.mk all     (from oracle/; build() runs it after the Makefile)
#     _ref/ref_afish               unmodified main.cpp + ref_afish.cpp: the `afish` record of the reference (CPU solver)
#     _ref/ref_afish_amrresident   the same record of the device-resident form (dropin/amr_resident_*.inc, as in the
#                                  Makefile's ref_amrresident) — the comparison point of tools/bench_reference_loop.py
#     _ref/ref_harness_amrdevice   the device form (dropin/amr_device_*.inc and amr_resident_udef.inc): every field-sized
#                                  phase of the body step on one cup2d_amr context, the same record
# As in the Makefile, main.cpp is spliced BY LINE NUMBER into a build intermediate under _ref/ that is deleted after use, and
# LIBDIR / LIBNAME / RPATH select the library (the product, or tests/host_emu's emulated build of it).
REF ?= /root/reference
OUT = _ref
CXX = /usr/bin/g++
CXXFLAGS = -O3 -fopenmp -std=c++17 -D_BS_=8 -include cfloat -Ishim -I$(REF) -w
LIBDIR ?= ../cup2d_b200
LIBNAME ?= cup2d_b200
RPATH ?= '$$ORIGIN/../../cup2d_b200'
AMRDEVICE ?= ref_harness_amrdevice
AFISH_RESIDENT ?= ref_afish_amrresident

all: afish afish_amrresident ref_amrdevice
afish: $(OUT)/ref_afish
afish_amrresident: $(OUT)/$(AFISH_RESIDENT)
ref_amrdevice: $(OUT)/$(AMRDEVICE)

$(OUT)/ref_spmat_cpu_afish.o: ref_spmat_cpu.cpp shim/mpi.h
	mkdir -p $(OUT)
	$(CXX) $(CXXFLAGS) -c ref_spmat_cpu.cpp -o $@

$(OUT)/ref_afish: ref_afish.cpp $(OUT)/ref_spmat_cpu_afish.o shim/mpi.h shim/gsl/gsl_linalg.h $(REF)/main.cpp amrdevice.mk
	$(CXX) $(CXXFLAGS) -c ref_afish.cpp -o $(OUT)/ref_afish.o
	$(CXX) -fopenmp -o $@ $(OUT)/ref_afish.o $(OUT)/ref_spmat_cpu_afish.o

$(OUT)/$(AFISH_RESIDENT): ref_afish.cpp $(OUT)/ref_spmat_cpu_afish.o $(REF)/main.cpp $(wildcard ../dropin/amr_resident_*.inc) \
                          ../dropin/b200_loop_glue.h shim/mpi.h amrdevice.mk
	sed -e '4658r ../dropin/amr_resident_tags.inc' -e '4660r ../dropin/amr_resident_tags_end.inc' \
	    -e '6607,6642d' -e '6606r ../dropin/amr_resident_rk2.inc' -e '6648,6679d' -e '6647r ../dropin/amr_resident_integrals.inc' \
	    -e '6945,6979d' -e '6944r ../dropin/amr_resident_blend.inc' \
	    -e '6981,7187d' -e '6980r ../dropin/amr_resident_udef.inc' -e '6980r ../dropin/amr_resident_pressure.inc' \
	    $(REF)/main.cpp > $(OUT)/main_afish_amrresident.cpp
	test `grep -c 'cup2d_b200' $(OUT)/main_afish_amrresident.cpp` -ge 7   # every fragment landed
	$(CXX) $(CXXFLAGS) -I../include -I$(OUT) -DCUP2D_PATCHED_MAIN=4 -include ../dropin/b200_loop_glue.h -c ref_afish.cpp -o $(OUT)/$(AFISH_RESIDENT).o
	rm -f $(OUT)/main_afish_amrresident.cpp
	$(CXX) -fopenmp -o $@ $(OUT)/$(AFISH_RESIDENT).o $(OUT)/ref_spmat_cpu_afish.o -L$(LIBDIR) -l$(LIBNAME) -Wl,-rpath,$(RPATH)

# main.cpp line ranges replaced (fragment): 4019-4024 (init: the context at the first ongrid, the only field upload),
# 4208-4467 and 4469-4556 (ongrid: rasterisation, surface normals, M / J / centre of mass / d_gm), 4659-4660 (tags),
# after 6544 and 6604 (regrid: adapt()'s new mesh in place), 6548-6575 (blend0: u_def assembly + cup2d_amr_udef_blend),
# 6585-6591 (umax), 6601 (dump), 6607-6642 (rk2), 6648-6679 (integrals), 6705-6943 (collide), 6945-6979 (penalize),
# 6981-7284 (amr_resident_udef, pressure, forces)
$(OUT)/$(AMRDEVICE): ref_afish.cpp $(OUT)/ref_spmat_cpu_afish.o $(REF)/main.cpp $(wildcard ../dropin/amr_device_*.inc) \
                     ../dropin/amr_resident_udef.inc ../dropin/b200_loop_glue.h shim/mpi.h amrdevice.mk
	sed -e '4019,4024d' -e '4018r ../dropin/amr_device_init.inc' -e '4208,4467d' \
	    -e '4469,4556d' -e '4468r ../dropin/amr_device_ongrid.inc' -e '4659,4660d' -e '4658r ../dropin/amr_device_tags.inc' \
	    -e '6544r ../dropin/amr_device_regrid.inc' -e '6548,6575d' -e '6547r ../dropin/amr_device_blend0.inc' \
	    -e '6585,6591d' -e '6584r ../dropin/amr_device_umax.inc' -e '6601d' -e '6600r ../dropin/amr_device_dump.inc' \
	    -e '6604r ../dropin/amr_device_regrid.inc' -e '6607,6642d' -e '6606r ../dropin/amr_device_rk2.inc' \
	    -e '6648,6679d' -e '6647r ../dropin/amr_device_integrals.inc' -e '6705,6943d' -e '6704r ../dropin/amr_device_collide.inc' \
	    -e '6945,6979d' -e '6944r ../dropin/amr_device_penalize.inc' -e '6981,7284d' -e '6980r ../dropin/amr_resident_udef.inc' \
	    -e '6980r ../dropin/amr_device_pressure.inc' -e '6980r ../dropin/amr_device_forces.inc' \
	    $(REF)/main.cpp > $(OUT)/main_amrdevice.cpp
	test `grep -c 'cup2d_b200' $(OUT)/main_amrdevice.cpp` -ge 15   # every fragment landed
	$(CXX) $(CXXFLAGS) -I../include -I$(OUT) -DCUP2D_PATCHED_MAIN=5 -include ../dropin/b200_loop_glue.h -c ref_afish.cpp -o $(OUT)/$(AMRDEVICE).o
	rm -f $(OUT)/main_amrdevice.cpp
	$(CXX) -fopenmp -o $@ $(OUT)/$(AMRDEVICE).o $(OUT)/ref_spmat_cpu_afish.o -L$(LIBDIR) -l$(LIBNAME) -Wl,-rpath,$(RPATH)

.PHONY: all afish afish_amrresident ref_amrdevice
