#!/bin/bash
# build.sh -- compiles the product library for sm_90a (nvcc cross-compiles without a GPU).
#   erasor_b200/_lib/liberasor_b200.so            the C-ABI library (include/erasor_b200.h)
#   erasor_b200/_lib/liberasor_b200_hostcheck.so  host-only build of binning.h, pcd_codec.h, pcd_binary.h, lzf_encode.h, bag_index.h, lz4_frame.h and bz2_stream.h for the CPU test-suite
set -euo pipefail
cd "$(dirname "$0")"
mkdir -p ../_lib ../_build
NVCC=${NVCC:-nvcc}
ARCH="-gencode arch=compute_90a,code=sm_90a"
# host float math (pose / inverse matrices) must not be FMA-contracted: the oracle restates it without (aarch64 g++ contracts by default)
CXXF="-O3 -std=c++17 -lineinfo -Xcompiler -fPIC -Xcompiler -ffp-contract=off"
$NVCC $ARCH $CXXF -Xptxas -v -c kernels.cu -o ../_build/kernels.o 2> ../_build/kernels.ptxas.log || { cat ../_build/kernels.ptxas.log; exit 1; }
$NVCC $ARCH $CXXF -Xptxas -v -c k1_geo.cu -o ../_build/k1_geo.o 2> ../_build/k1_geo.ptxas.log || { cat ../_build/k1_geo.ptxas.log; exit 1; }
$NVCC $ARCH $CXXF -c erasor_capi.cu -o ../_build/erasor_capi.o
$NVCC $ARCH $CXXF -Xptxas -v -c updater_kernels.cu -o ../_build/updater_kernels.o 2> ../_build/updater_kernels.ptxas.log || { cat ../_build/updater_kernels.ptxas.log; exit 1; }
$NVCC $ARCH $CXXF -c updater_capi.cu -o ../_build/updater_capi.o
$NVCC $ARCH $CXXF -c mapgen_capi.cu -o ../_build/mapgen_capi.o
$NVCC $ARCH $CXXF -Xptxas -v -c eval_kernels.cu -o ../_build/eval_kernels.o 2> ../_build/eval_kernels.ptxas.log || { cat ../_build/eval_kernels.ptxas.log; exit 1; }
$NVCC $ARCH $CXXF -Xptxas -v -c pcd_kernels.cu -o ../_build/pcd_kernels.o 2> ../_build/pcd_kernels.ptxas.log || { cat ../_build/pcd_kernels.ptxas.log; exit 1; }
$NVCC $ARCH $CXXF -Xptxas -v -c voxelize_batch.cu -o ../_build/voxelize_batch.o 2> ../_build/voxelize_batch.ptxas.log || { cat ../_build/voxelize_batch.ptxas.log; exit 1; }
g++ -O2 -std=c++17 -fPIC -ffp-contract=off -c binning_tables.cpp -o ../_build/binning_tables.o
$NVCC $ARCH -shared -o ../_lib/liberasor_b200.so ../_build/kernels.o ../_build/k1_geo.o ../_build/erasor_capi.o ../_build/updater_kernels.o ../_build/updater_capi.o ../_build/mapgen_capi.o ../_build/eval_kernels.o ../_build/pcd_kernels.o ../_build/voxelize_batch.o ../_build/binning_tables.o -lquadmath -lcudart -ldl
g++ -O2 -std=c++17 -fPIC -shared -ffp-contract=off -I/usr/local/cuda/include -o ../_lib/liberasor_b200_hostcheck.so host_selftest.cpp binning_tables.cpp -lquadmath
g++ -std=c++17 -O2 -I/usr/local/cuda/include -o ../_lib/offline_map_updater_main ../../examples/offline_map_updater_main.cpp -L../_lib -lerasor_b200 -Wl,-rpath,'$ORIGIN' \
    -L/usr/local/cuda/lib64 -Wl,-rpath,/usr/local/cuda/lib64 -lcudart
g++ -std=c++17 -O2 -I/usr/local/cuda/include -o ../_lib/mapgen_main ../../examples/mapgen_main.cpp -L../_lib -lerasor_b200 -Wl,-rpath,'$ORIGIN' \
    -L/usr/local/cuda/lib64 -Wl,-rpath,/usr/local/cuda/lib64 -lcudart
g++ -std=c++17 -O2 -I/usr/local/cuda/include -o ../_lib/static_map_nodes_main ../../examples/static_map_nodes_main.cpp -L../_lib -lerasor_b200 -Wl,-rpath,'$ORIGIN' \
    -L/usr/local/cuda/lib64 -Wl,-rpath,/usr/local/cuda/lib64 -lcudart
echo "built: $(ls ../_lib)"
# C++ host-class demo (include/erasor/erasor.hpp over the C ABI)
g++ -std=c++17 -O2 -o ../_lib/erasor_cpp_demo ../../examples/erasor_cpp_demo.cpp -L../_lib -lerasor_b200 -Wl,-rpath,'$ORIGIN' \
    -L/usr/local/cuda/lib64 -Wl,-rpath,/usr/local/cuda/lib64
# micro-benchmark of __match_any_sync latency and throughput (the voxelisation kernel groups equal keys with it)
$NVCC $ARCH -O3 -o ../_lib/mb_match ../../scripts/mb_match.cu
