#!/bin/bash
# Compares the SASS of every kernel of a previous build (git ref, default HEAD) with the working tree's build: prints
# "<diff lines> <instructions> <kernel>" per kernel of every translation unit of the old build.  0 diff lines = byte-identical code.  Used to prove that an
# opt-in template variant leaves the hardware-verified default kernels untouched (renamed instantiations: pass a sed script).
#   scratch/sass_diff.sh [ref] ['s/old-mangled-suffix/new-mangled-suffix/;...']
set -e
REF=${1:-HEAD}; MAP=${2:-}
ROOT=$(cd "$(dirname "$0")/.." && pwd); T=$(mktemp -d)
git -C "$ROOT" archive "$REF" online-3d-bpp-pct_b200/csrc include | tar -x -C "$T"
FLAGS="-O3 -std=c++17 -lineinfo -fmad=false -Xcompiler -fPIC -I$T/include -I$T/online-3d-bpp-pct_b200/csrc -gencode arch=compute_90a,code=sm_90a"
norm() { grep -E "^\s+/\*[0-9a-f]{4,6}\*/" | sed 's#/\*[0-9a-f]*\*/##'; }
UNITS=$(cd "$T/online-3d-bpp-pct_b200/csrc" && ls *.cu | sed 's/\.cu$//')  # every translation unit of the old build
for u in $UNITS; do nvcc $FLAGS -c "$T/online-3d-bpp-pct_b200/csrc/$u.cu" -o "$T/$u.o" & done
for j in $(jobs -p); do wait "$j"; done
for u in $UNITS; do
  NEW="$ROOT/online-3d-bpp-pct_b200/csrc/$u.o"
  cuobjdump -sass "$NEW" | grep "Function :" | awk '{print $3}' > "$T/new.txt"
  for f in $(cuobjdump -sass "$T/$u.o" | grep "Function :" | awk '{print $3}'); do
    g=$f
    grep -qx "$g" "$T/new.txt" || { [ -n "$MAP" ] && g=$(echo "$f" | sed "$MAP"); }
    grep -qx "$g" "$T/new.txt" || { echo "MISSING - $f"; continue; }
    cuobjdump -sass -fun "$f" "$T/$u.o" | norm > "$T/a.txt"
    cuobjdump -sass -fun "$g" "$NEW" | norm > "$T/b.txt"
    echo "$(diff "$T/a.txt" "$T/b.txt" | wc -l) $(wc -l < "$T/a.txt") $f"
  done
done
rm -rf "$T"
