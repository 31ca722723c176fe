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

$(LIB): $(OBJDIR)/kernels_f32.o $(OBJDIR)/kernels_vx.o $(OBJDIR)/kernels_f64.o $(OBJDIR)/film.o $(OBJDIR)/api.o $(OBJDIR)/kdbuild.o $(OBJDIR)/bvhbuild.o $(OBJDIR)/objparse.o
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
hostemu: $(HOSTEMU)
$(HOSTEMU): tests/hostemu/hostemu.cu $(CSRC)/kdbuild.cpp $(CSRC)/bvhbuild.cpp $(HDRS)
	@mkdir -p $(dir $@)
	nvcc -std=c++17 -O2 -DRPTB_HOST_EMU -DRPTB_BUILD_BVH8=1 -DRPTB_BUILD_BVH4=1 -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC,-fopenmp,-ffp-contract=off -shared -Xlinker -Bsymbolic -o $@ tests/hostemu/hostemu.cu $(CSRC)/kdbuild.cpp $(CSRC)/bvhbuild.cpp -lgomp

clean:
	rm -rf build $(LIB) $(ORACLE) tests/hostemu/_build
.PHONY: all lib oracle examples hostemu clean
