#!/bin/bash
# scratch/mkvariant.sh NAME "-DF2_MINB=12 ..."  -> scratch/variants/lib_NAME.so (pct_discrete.cu recompiled with the defines; other objects reused)
set -e
cd "$(dirname "$0")/../online-3d-bpp-pct_b200/csrc"
N=$1; shift
mkdir -p ../../scratch/variants
nvcc -O3 -std=c++17 -lineinfo -fmad=false -Xcompiler -fPIC -I../../include -I. -gencode arch=compute_90a,code=sm_90a "$@" -c pct_discrete.cu -o ../../scratch/variants/pct_discrete_$N.o
nvcc -shared -gencode arch=compute_90a,code=sm_90a -o ../../scratch/variants/lib_$N.so ../../scratch/variants/pct_discrete_$N.o pct_continuous.o pct_api.o -cudart static
echo built lib_$N.so
