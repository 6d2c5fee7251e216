#!/bin/bash
# Build a variant of the library with extra -D options (in-tree, git-ignored):
#   scripts/build_variant.sh dw3 -DSYN_DW3=1      -> synergynet_b200/libsynergy_b200_var_dw3.so
# then, on the GPU machine:
#   SYN_LIB_PATH=$PWD/synergynet_b200/libsynergy_b200_var_dw3.so python scripts/quick_variant_check.py
#   SYN_LIB_PATH=...                                            python -m pytest tests/test_gpu_parity.py -q
set -e
name=$1; shift
cd "$(dirname "$0")/.."
nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -shared "$@" -Iinclude \
     -o synergynet_b200/libsynergy_b200_var_$name.so synergynet_b200/csrc/synergy_b200.cu
echo "built synergynet_b200/libsynergy_b200_var_$name.so ($*)"
