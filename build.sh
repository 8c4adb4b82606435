#!/bin/bash
# Build libvbert_b200.so for sm_90a (in-tree; the .so is git-ignored).
set -e
make -C "$(dirname "$0")/visualbert_b200/csrc" -j"$(nproc)" "$@"
