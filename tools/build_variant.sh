#!/bin/bash
# A/B helper: build a variant of libcupoch_b200.so with extra -D flags for icp.cu into build_variants/<name>.so
# usage: tools/build_variant.sh name -DICP_MIN_BLOCKS=8
set -e
cd "$(dirname "$0")/.."
name=$1; shift
mkdir -p build_variants /tmp/cphb_var_$name
python -m cupoch_b200.build >/dev/null
S=cupoch_b200/csrc
nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -fmad=false -Xcompiler -fPIC -Iinclude -I$S "$@" -c $S/icp.cu -o /tmp/cphb_var_$name/icp.o
objs=$(for f in index sort search voxel features filters voxelgrid comm reduce fpfh cluster occgrid; do echo $S/_build/$f.o; done)
nvcc -shared -o build_variants/$name.so $objs /tmp/cphb_var_$name/icp.o -cudart static -ldl -gencode arch=compute_90a,code=sm_90a
echo build_variants/$name.so
