#!/bin/bash
# Builds libvpt_b200.so (the product) in-tree for sm_90a (H100).  nvcc cross-compiles without a GPU.
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
OUT="$HERE/../lib"
mkdir -p "$OUT" "$HERE/_obj"
ARCH="-gencode arch=compute_90a,code=sm_90a"
NVCC="${NVCC:-nvcc}"
# kernels: the reference's numeric flags (--use_fast_math) so per-seed parity is reachable
$NVCC $ARCH -O3 --use_fast_math -lineinfo -std=c++17 -Xcompiler -fPIC ${VPT_KERNEL_DEFS:-} -c "$HERE/device/vpt_kernels.cu" -o "$HERE/_obj/vpt_kernels.o"
$NVCC $ARCH -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -c "$HERE/device/vpt_bricks.cu" -o "$HERE/_obj/vpt_bricks.o"
# denoiser: the same flags as vpt_kernels.cu, so its display words come out of the very same tonemap code as k_resolve's
$NVCC $ARCH -O3 --use_fast_math -lineinfo -std=c++17 -Xcompiler -fPIC -c "$HERE/device/vpt_denoise.cu" -o "$HERE/_obj/vpt_denoise.o"
# temporal filter: the same flags again, so its blend is accum's running-mean arithmetic and its display words k_resolve's, bit for bit
$NVCC $ARCH -O3 --use_fast_math -lineinfo -std=c++17 -Xcompiler -fPIC -c "$HERE/device/vpt_temporal.cu" -o "$HERE/_obj/vpt_temporal.o"
$NVCC $ARCH -O3 --use_fast_math -lineinfo -std=c++17 -Xcompiler -fPIC -c "$HERE/device/vpt_bruneton.cu" -o "$HERE/_obj/vpt_bruneton.o"
# octree build: plain IEEE flags, as the reference's bvh object
$NVCC $ARCH -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-ffp-contract=off -c "$HERE/device/vpt_octree.cu" -o "$HERE/_obj/vpt_octree.o"
$NVCC $ARCH -O2 -std=c++17 -Xcompiler -fPIC,-ffp-contract=off ${VPT_KERNEL_DEFS:-} -x cu -c "$HERE/host/vpt_context.cpp" -o "$HERE/_obj/vpt_context.o"
$NVCC $ARCH -O2 -std=c++17 -Xcompiler -fPIC,-ffp-contract=off -x cu -c "$HERE/host/vpt_scene_build.cpp" -o "$HERE/_obj/vpt_scene_build.o"
g++ -O2 -std=c++17 -fPIC -c "$HERE/host/vdb_reader.cpp" -o "$HERE/_obj/vdb_reader.o"
g++ -O2 -std=c++17 -fPIC -c "$HERE/host/image_io.cpp" -o "$HERE/_obj/image_io.o"
g++ -O2 -std=c++17 -fPIC -ffp-contract=off -c "$HERE/host/sky_table.cpp" -o "$HERE/_obj/sky_table.o"
# level (A): the single-entry module for the reference's unchanged Driver-API loader (cuModuleLoad -> "volume_rt_kernel")
$NVCC $ARCH -cubin -O3 --use_fast_math -lineinfo -std=c++17 -DVPT_LEVEL_A_MODULE "$HERE/device/vpt_level_a.cu" -o "$OUT/.volume_rt_kernel_b200.cubin.tmp"
mv -f "$OUT/.volume_rt_kernel_b200.cubin.tmp" "$OUT/volume_rt_kernel_b200.cubin"
LIBNAME="${VPT_LIB_NAME:-libvpt_b200.so}"
$NVCC $ARCH -O2 -std=c++17 -Xcompiler -fPIC,-ffp-contract=off -x cu -c "$HERE/host/vpt_atmosphere_host.cpp" -o "$HERE/_obj/vpt_atmosphere_host.o"
$NVCC $ARCH -O2 -std=c++17 -Xcompiler -fPIC -x cu -c "$HERE/host/vpt_comm.cpp" -o "$HERE/_obj/vpt_comm.o"
# link under a temporary name and rename: a snapshot (gpurun) taken during the build never sees a half-written library
$NVCC $ARCH -shared -o "$OUT/.$LIBNAME.tmp" "$HERE"/_obj/*.o -lz -ldl
mv -f "$OUT/.$LIBNAME.tmp" "$OUT/$LIBNAME"
echo "built $OUT/$LIBNAME"
