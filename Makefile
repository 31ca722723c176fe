# Builds the CUDA library (product) and the CPU oracle (test infrastructure).
#   make            -> rpt_b200/lib/librpt_b200.so + oracle/_build/liboracle.so
#   make lib        -> product only
#   make oracle     -> oracle only
NVCC      ?= nvcc
CXX       := g++
ARCH      := -gencode arch=compute_90a,code=sm_90a
NVFLAGS   := -std=c++17 -O3 -lineinfo $(ARCH) -Xcompiler -fPIC,-fopenmp -Xptxas -v
CSRC      := rpt_b200/csrc
OBJDIR    := build/obj
LIB       := rpt_b200/lib/librpt_b200.so
ORACLE    := oracle/_build/liboracle.so
HDRS      := $(wildcard $(CSRC)/*.cuh) $(wildcard $(CSRC)/*.h) include/rpt_b200.h

all: lib oracle
lib: $(LIB)
oracle: $(ORACLE)

# the f32 product path: SFU approximations for divide/sqrt/exp/log (|rel err| ~ 1e-6, far
# inside the f32 parity tolerance), denormals flushed
$(OBJDIR)/kernels_f32.o: $(CSRC)/kernels_f32.cu $(HDRS)
	@mkdir -p $(OBJDIR)
	$(NVCC) $(NVFLAGS) --use_fast_math -c $< -o $@ 2> $(OBJDIR)/kernels_f32.ptxas.log || (cat $(OBJDIR)/kernels_f32.ptxas.log; false)
$(OBJDIR)/kernels_vx.o: $(CSRC)/kernels_vx.cu $(HDRS)
	@mkdir -p $(OBJDIR)
	$(NVCC) $(NVFLAGS) --use_fast_math -c $< -o $@ 2> $(OBJDIR)/kernels_vx.ptxas.log || (cat $(OBJDIR)/kernels_vx.ptxas.log; false)
# the parity gate keeps products and sums separately rounded, like the reference's f64 code
$(OBJDIR)/kernels_f64.o: $(CSRC)/kernels_f64.cu $(HDRS)
	@mkdir -p $(OBJDIR)
	$(NVCC) $(NVFLAGS) -fmad=false -c $< -o $@ 2> $(OBJDIR)/kernels_f64.ptxas.log || (cat $(OBJDIR)/kernels_f64.ptxas.log; false)
# the adaptive criterion (adaptive.h) rounds every operation on its own, like its numpy and host-emulation restatements
$(OBJDIR)/adaptive.o: $(CSRC)/adaptive.cu $(HDRS)
	@mkdir -p $(OBJDIR)
	$(NVCC) $(NVFLAGS) -fmad=false -c $< -o $@ 2> $(OBJDIR)/adaptive.ptxas.log || (cat $(OBJDIR)/adaptive.ptxas.log; false)
# the denoiser (denoise.h) likewise: its numpy restatement and host emulation round every operation on its own
$(OBJDIR)/denoise.o: $(CSRC)/denoise.cu $(HDRS)
	@mkdir -p $(OBJDIR)
	$(NVCC) $(NVFLAGS) -fmad=false -c $< -o $@ 2> $(OBJDIR)/denoise.ptxas.log || (cat $(OBJDIR)/denoise.ptxas.log; false)
# the reprojection (reproject.h) likewise: its numpy restatement and host emulation round every operation on its own
$(OBJDIR)/reproject.o: $(CSRC)/reproject.cu $(HDRS)
	@mkdir -p $(OBJDIR)
	$(NVCC) $(NVFLAGS) -fmad=false -c $< -o $@ 2> $(OBJDIR)/reproject.ptxas.log || (cat $(OBJDIR)/reproject.ptxas.log; false)
# the guided criterion (guided.h) likewise: its numpy restatement and host emulation round every operation on its own
$(OBJDIR)/guided.o: $(CSRC)/guided.cu $(HDRS)
	@mkdir -p $(OBJDIR)
	$(NVCC) $(NVFLAGS) -fmad=false -c $< -o $@ 2> $(OBJDIR)/guided.ptxas.log || (cat $(OBJDIR)/guided.ptxas.log; false)
# the error estimate from two half buffers (halves.h) likewise: its numpy restatement and host emulation round every
# operation on its own
$(OBJDIR)/halves.o: $(CSRC)/halves.cu $(HDRS)
	@mkdir -p $(OBJDIR)
	$(NVCC) $(NVFLAGS) -fmad=false -c $< -o $@ 2> $(OBJDIR)/halves.ptxas.log || (cat $(OBJDIR)/halves.ptxas.log; false)
# the per-pixel choice of the filter's pass count (select.h) likewise: its numpy restatement and host emulation round
# every operation on its own
$(OBJDIR)/select.o: $(CSRC)/select.cu $(HDRS)
	@mkdir -p $(OBJDIR)
	$(NVCC) $(NVFLAGS) -fmad=false -c $< -o $@ 2> $(OBJDIR)/select.ptxas.log || (cat $(OBJDIR)/select.ptxas.log; false)
# the cross-filtered denoiser with a smoothed selection map (cross.h) likewise: its numpy restatement and host emulation
# round every operation on its own
$(OBJDIR)/cross.o: $(CSRC)/cross.cu $(HDRS)
	@mkdir -p $(OBJDIR)
	$(NVCC) $(NVFLAGS) -fmad=false -c $< -o $@ 2> $(OBJDIR)/cross.ptxas.log || (cat $(OBJDIR)/cross.ptxas.log; false)
# the delta exchange (delta.h) only moves doubles; compiled like its neighbours all the same
$(OBJDIR)/delta.o: $(CSRC)/delta.cu $(HDRS)
	@mkdir -p $(OBJDIR)
	$(NVCC) $(NVFLAGS) -fmad=false -c $< -o $@ 2> $(OBJDIR)/delta.ptxas.log || (cat $(OBJDIR)/delta.ptxas.log; false)
$(OBJDIR)/film.o: $(CSRC)/film.cu $(HDRS)
	@mkdir -p $(OBJDIR)
	$(NVCC) $(NVFLAGS) -c $< -o $@ 2> $(OBJDIR)/film.ptxas.log || (cat $(OBJDIR)/film.ptxas.log; false)
$(OBJDIR)/api.o: $(CSRC)/api.cu $(HDRS)
	@mkdir -p $(OBJDIR)
	$(NVCC) $(NVFLAGS) -c $< -o $@ 2> $(OBJDIR)/api.ptxas.log || (cat $(OBJDIR)/api.ptxas.log; false)
$(OBJDIR)/kdbuild.o: $(CSRC)/kdbuild.cpp include/rpt_b200.h
	@mkdir -p $(OBJDIR)
	$(CXX) -std=c++17 -O3 -fPIC -fopenmp -Wall -c $< -o $@
$(OBJDIR)/bvhbuild.o: $(CSRC)/bvhbuild.cpp $(CSRC)/scene_dev.cuh $(CSRC)/vec.cuh
	@mkdir -p $(OBJDIR)
	$(CXX) -std=c++17 -O3 -fPIC -fopenmp -Wall -I/usr/local/cuda/include -c $< -o $@
$(OBJDIR)/objparse.o: $(CSRC)/objparse.cpp
	@mkdir -p $(OBJDIR)
	$(CXX) -std=c++17 -O3 -fPIC -Wall -c $< -o $@

$(LIB): $(OBJDIR)/kernels_f32.o $(OBJDIR)/kernels_vx.o $(OBJDIR)/kernels_f64.o $(OBJDIR)/film.o $(OBJDIR)/adaptive.o $(OBJDIR)/denoise.o $(OBJDIR)/guided.o $(OBJDIR)/halves.o $(OBJDIR)/select.o $(OBJDIR)/cross.o $(OBJDIR)/delta.o $(OBJDIR)/reproject.o $(OBJDIR)/api.o $(OBJDIR)/kdbuild.o $(OBJDIR)/bvhbuild.o $(OBJDIR)/objparse.o
	@mkdir -p rpt_b200/lib
	$(NVCC) -shared $(ARCH) -o $@ $^ -Xcompiler -fopenmp -lgomp -cudart shared

# -march=x86-64-v3: AVX2 hosts; no FMA contraction so
# the f64 arithmetic rounds like the reference's
$(ORACLE): oracle/oracle.cpp include/rpt_b200.h
	@mkdir -p oracle/_build
	$(CXX) -std=c++17 -O3 -march=x86-64-v3 -ffp-contract=off -fopenmp -fPIC -shared -Wall -Wextra -o $@ $<

# C++ host mirror example (needs a GPU to run)
examples: build/sphere_cpp build/fractal_spheres_cpp
build/%_cpp: examples/%.cpp include/rpt.hpp include/rpt_b200.h $(LIB)
	$(CXX) -std=c++17 -O2 -Wall -o $@ $< -Lrpt_b200/lib -lrpt_b200 -Wl,-rpath,'$$ORIGIN/../rpt_b200/lib'

# test infrastructure: the device geometry functions compiled for the host (tests/hostemu/hostemu.cu).  -Bsymbolic: the
# library is loaded next to librpt_b200.so (RTLD_GLOBAL), whose copies of the inline flatteners were compiled with other
# switches (RPTB_BUILD_BVH8) -- hostemu must call its own
HOSTEMU := tests/hostemu/_build/libhostemu.so
# the same emulation plus adaptive sampling's list-scheduled megakernel and convergence test (tests/hostemu/hostemu_list.cu)
HOSTEMU_LIST := tests/hostemu/_build/libhostemu_list.so
# the same emulation plus the feature pass (features.cuh) and the denoiser's per-pixel functions (tests/hostemu/hostemu_denoise.cu)
HOSTEMU_DENOISE := tests/hostemu/_build/libhostemu_denoise.so
# the same emulation plus the renders given no counters (the packed-table F_NOCOUNT twins; tests/hostemu/hostemu_slim.cu)
HOSTEMU_SLIM := tests/hostemu/_build/libhostemu_slim.so
# the denoiser's emulation plus the reprojection's per-pixel function (reproject.h; tests/hostemu/hostemu_reproject.cu) and
# its per-element form for a shard's compact tiles (tests/hostemu/hostemu_reproject_part.cu), and the history test of
# the merge, per pixel and per element (tests/hostemu/hostemu_reproject_merge.cu), and the history halves of both
# (tests/hostemu/hostemu_reproject_halves.cu)
HOSTEMU_REPROJECT := tests/hostemu/_build/libhostemu_reproject.so
# the denoiser's emulation plus the guided adaptive criterion, per pixel and per slot of a part (guided.h;
# tests/hostemu/hostemu_guided.cu)
HOSTEMU_GUIDED := tests/hostemu/_build/libhostemu_guided.so
# the delta exchange's per-element export and import (delta.h; tests/hostemu/hostemu_delta.cu)
HOSTEMU_DELTA := tests/hostemu/_build/libhostemu_delta.so
# the same for the delta block of a shard with halves (delta.h; tests/hostemu/hostemu_delta_halves.cu)
HOSTEMU_DELTA_HALVES := tests/hostemu/_build/libhostemu_delta_halves.so
# the error estimate's per-pixel functions (halves.h; tests/hostemu/hostemu_halves.cu)
HOSTEMU_HALVES := tests/hostemu/_build/libhostemu_halves.so
# the choice of the filter's pass count per pixel (select.h; tests/hostemu/hostemu_select.cu)
HOSTEMU_SELECT := tests/hostemu/_build/libhostemu_select.so
# the cross-filtered denoiser's per-pixel functions (cross.h; tests/hostemu/hostemu_cross.cu)
HOSTEMU_CROSS := tests/hostemu/_build/libhostemu_cross.so
hostemu: $(HOSTEMU) $(HOSTEMU_LIST) $(HOSTEMU_DENOISE) $(HOSTEMU_SLIM) $(HOSTEMU_REPROJECT) $(HOSTEMU_GUIDED) $(HOSTEMU_DELTA) $(HOSTEMU_DELTA_HALVES) $(HOSTEMU_HALVES) $(HOSTEMU_SELECT) $(HOSTEMU_CROSS)
$(HOSTEMU): tests/hostemu/hostemu.cu $(CSRC)/kdbuild.cpp $(CSRC)/bvhbuild.cpp $(HDRS)
	@mkdir -p $(dir $@)
	nvcc -std=c++17 -O2 -DRPTB_HOST_EMU -DRPTB_BUILD_BVH8=1 -DRPTB_BUILD_BVH4=1 -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC,-fopenmp,-ffp-contract=off -shared -Xlinker -Bsymbolic -o $@ tests/hostemu/hostemu.cu $(CSRC)/kdbuild.cpp $(CSRC)/bvhbuild.cpp -lgomp
$(HOSTEMU_LIST): tests/hostemu/hostemu_list.cu tests/hostemu/hostemu.cu $(CSRC)/kdbuild.cpp $(CSRC)/bvhbuild.cpp $(HDRS)
	@mkdir -p $(dir $@)
	nvcc -std=c++17 -O2 -DRPTB_HOST_EMU -DRPTB_BUILD_BVH8=1 -DRPTB_BUILD_BVH4=1 -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC,-fopenmp,-ffp-contract=off -shared -Xlinker -Bsymbolic -o $@ tests/hostemu/hostemu_list.cu $(CSRC)/kdbuild.cpp $(CSRC)/bvhbuild.cpp -lgomp
$(HOSTEMU_DENOISE): tests/hostemu/hostemu_denoise.cu tests/hostemu/hostemu.cu $(CSRC)/kdbuild.cpp $(CSRC)/bvhbuild.cpp $(HDRS)
	@mkdir -p $(dir $@)
	nvcc -std=c++17 -O2 -DRPTB_HOST_EMU -DRPTB_BUILD_BVH8=1 -DRPTB_BUILD_BVH4=1 -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC,-fopenmp,-ffp-contract=off -shared -Xlinker -Bsymbolic -o $@ tests/hostemu/hostemu_denoise.cu $(CSRC)/kdbuild.cpp $(CSRC)/bvhbuild.cpp -lgomp
$(HOSTEMU_SLIM): tests/hostemu/hostemu_slim.cu tests/hostemu/hostemu.cu $(CSRC)/kdbuild.cpp $(CSRC)/bvhbuild.cpp $(HDRS)
	@mkdir -p $(dir $@)
	nvcc -std=c++17 -O2 -DRPTB_HOST_EMU -DRPTB_BUILD_BVH8=1 -DRPTB_BUILD_BVH4=1 -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC,-fopenmp,-ffp-contract=off -shared -Xlinker -Bsymbolic -o $@ tests/hostemu/hostemu_slim.cu $(CSRC)/kdbuild.cpp $(CSRC)/bvhbuild.cpp -lgomp
$(HOSTEMU_REPROJECT): tests/hostemu/hostemu_reproject.cu tests/hostemu/hostemu_reproject_part.cu tests/hostemu/hostemu_reproject_merge.cu tests/hostemu/hostemu_reproject_halves.cu tests/hostemu/hostemu_denoise.cu tests/hostemu/hostemu.cu $(CSRC)/kdbuild.cpp $(CSRC)/bvhbuild.cpp $(HDRS)
	@mkdir -p $(dir $@)
	nvcc -std=c++17 -O2 -DRPTB_HOST_EMU -DRPTB_BUILD_BVH8=1 -DRPTB_BUILD_BVH4=1 -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC,-fopenmp,-ffp-contract=off -shared -Xlinker -Bsymbolic -o $@ tests/hostemu/hostemu_reproject.cu tests/hostemu/hostemu_reproject_part.cu tests/hostemu/hostemu_reproject_merge.cu tests/hostemu/hostemu_reproject_halves.cu $(CSRC)/kdbuild.cpp $(CSRC)/bvhbuild.cpp -lgomp
$(HOSTEMU_GUIDED): tests/hostemu/hostemu_guided.cu tests/hostemu/hostemu_denoise.cu tests/hostemu/hostemu.cu $(CSRC)/kdbuild.cpp $(CSRC)/bvhbuild.cpp $(HDRS)
	@mkdir -p $(dir $@)
	nvcc -std=c++17 -O2 -DRPTB_HOST_EMU -DRPTB_BUILD_BVH8=1 -DRPTB_BUILD_BVH4=1 -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC,-fopenmp,-ffp-contract=off -shared -Xlinker -Bsymbolic -o $@ tests/hostemu/hostemu_guided.cu $(CSRC)/kdbuild.cpp $(CSRC)/bvhbuild.cpp -lgomp
$(HOSTEMU_DELTA): tests/hostemu/hostemu_delta.cu $(HDRS)
	@mkdir -p $(dir $@)
	nvcc -std=c++17 -O2 -DRPTB_HOST_EMU -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC,-ffp-contract=off -shared -Xlinker -Bsymbolic -o $@ tests/hostemu/hostemu_delta.cu
$(HOSTEMU_DELTA_HALVES): tests/hostemu/hostemu_delta_halves.cu $(HDRS)
	@mkdir -p $(dir $@)
	nvcc -std=c++17 -O2 -DRPTB_HOST_EMU -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC,-ffp-contract=off -shared -Xlinker -Bsymbolic -o $@ tests/hostemu/hostemu_delta_halves.cu
$(HOSTEMU_HALVES): tests/hostemu/hostemu_halves.cu $(HDRS)
	@mkdir -p $(dir $@)
	nvcc -std=c++17 -O2 -DRPTB_HOST_EMU -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC,-fopenmp,-ffp-contract=off -shared -Xlinker -Bsymbolic -o $@ tests/hostemu/hostemu_halves.cu -lgomp
$(HOSTEMU_SELECT): tests/hostemu/hostemu_select.cu $(HDRS)
	@mkdir -p $(dir $@)
	nvcc -std=c++17 -O2 -DRPTB_HOST_EMU -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC,-fopenmp,-ffp-contract=off -shared -Xlinker -Bsymbolic -o $@ tests/hostemu/hostemu_select.cu -lgomp
$(HOSTEMU_CROSS): tests/hostemu/hostemu_cross.cu $(HDRS)
	@mkdir -p $(dir $@)
	nvcc -std=c++17 -O2 -DRPTB_HOST_EMU -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC,-fopenmp,-ffp-contract=off -shared -Xlinker -Bsymbolic -o $@ tests/hostemu/hostemu_cross.cu -lgomp

clean:
	rm -rf build $(LIB) $(ORACLE) tests/hostemu/_build
.PHONY: all lib oracle examples hostemu clean
