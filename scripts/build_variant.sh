#!/bin/bash
# Build a second copy of the library with extra compile flags, for A/B timing on one GPU in one process tree:
#   scripts/build_variant.sh noprefetch "-DSOME_MACRO=0"
#   VB_LIB_PATH=visualbert_b200/lib/libvbert_b200_noprefetch.so python bench.py --no-cpu-baseline
set -e
name=$1; shift
cd "$(dirname "$0")/../visualbert_b200/csrc"
make -j 16 OBJDIR=../lib/obj_$name LIB=../lib/libvbert_b200_$name.so EXTRA="$*"
