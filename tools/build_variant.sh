#!/bin/bash
# A/B builds of the f32 kernels: tools/build_variant.sh <tag> <extra nvcc flags...>
# -> rpt_b200/lib/librpt_b200_<tag>.so (select it with RPTB_LIB=...; everything but kernels_f32.o is shared with the main build)
set -e
tag=$1; shift
mkdir -p build/obj_$tag
nvcc -std=c++17 -O3 -lineinfo -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC,-fopenmp -Xptxas -v --use_fast_math "$@" \
  -c rpt_b200/csrc/kernels_f32.cu -o build/obj_$tag/kernels_f32.o 2> build/obj_$tag/kernels_f32.ptxas.log
nvcc -shared -gencode arch=compute_90a,code=sm_90a -o rpt_b200/lib/librpt_b200_$tag.so build/obj_$tag/kernels_f32.o build/obj/kernels_vx.o \
  build/obj/kernels_f64.o build/obj/film.o build/obj/api.o build/obj/kdbuild.o build/obj/bvhbuild.o build/obj/objparse.o -Xcompiler -fopenmp -lgomp -cudart shared
echo built rpt_b200/lib/librpt_b200_$tag.so
