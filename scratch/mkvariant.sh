#!/bin/bash
# scratch/mkvariant.sh NAME "-DK2_MINB=12 ..."  -> scratch/variants/lib_NAME.so (pct_discrete.cu recompiled with the defines, linked with the
# Makefile's other objects; run `make` in csrc first) for A/B runs through PCT_B200_LIB.  UNIT=pct_buffer recompiles that unit instead.
set -e
cd "$(dirname "$0")/../online-3d-bpp-pct_b200/csrc"
N=$1; shift
U=${UNIT:-pct_discrete}
OBJS=$(sed -n 's/^OBJS = //p' Makefile)
mkdir -p ../../scratch/variants
nvcc -O3 -std=c++17 -lineinfo -fmad=false -Xcompiler -fPIC -I../../include -I. -gencode arch=compute_90a,code=sm_90a $@ -c $U.cu -o ../../scratch/variants/${U}_$N.o
nvcc -shared -gencode arch=compute_90a,code=sm_90a -o ../../scratch/variants/lib_$N.so ../../scratch/variants/${U}_$N.o ${OBJS/$U.o/} -cudart static
echo built lib_$N.so
