#!/bin/bash
# Builds lidarslam_ros2_b200/csrc/libb200reg.so for sm_90a (H100), in-tree.
set -e
cd "$(dirname "$0")/lidarslam_ros2_b200/csrc"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -ccbin $(command -v g++) ${B200_NVCC_EXTRA}"
OBJS=""
for f in grid_index voxel_map ndt_solver ndt_aux ndt_score nn_grid voxelgrid gicp cloud_codec pcd_codec pcd_load deskew comm capi scanmatcher place_recognition occupancy static_map relocalize elevation consistency map_changes mesh octomap; do
  if [ ! -f $f.o ] || [ $f.cu -nt $f.o ] || [ -n "$(find . -name '*.cuh' -newer $f.o -o -name '*.hpp' -newer $f.o -o -name 'b200reg.h' -newer $f.o 2>/dev/null)" ] || [ ../../include/b200reg.h -nt $f.o ] || [ ../../include/b200comm.h -nt $f.o ]; then
    echo "nvcc $f.cu"
    # gicp.cu: no FMA contraction. The reference builds for baseline x86-64 (no FMA) and GICP's line search compares f32
    # cost values (gicp_omp_impl.hpp:264-270): a fused a*b+c changes them in the last bit, and the capped inner BFGS
    # (20 iterations) amplifies that to centimetres on weakly constrained scenes. The NDT kernels spell their un-fused
    # arithmetic out with __fmul_rn / __fadd_rn where parity needs it.
    EXTRA=""; [ $f = gicp ] && EXTRA="-fmad=false"
    # scanmatcher.cu: its host float arithmetic (csrc/sensor_frame.hpp) must match the un-fused device transform bit for bit
    [ $f = scanmatcher ] && EXTRA="-Xcompiler -ffp-contract=off"
    $NVCC $FLAGS $EXTRA -Xptxas -v -c $f.cu -o $f.o 2> $f.ptxas.log || { cat $f.ptxas.log; exit 1; }
  fi
  OBJS="$OBJS $f.o"
done
$NVCC -gencode arch=compute_90a,code=sm_90a -shared -o libb200reg.so $OBJS -ccbin $(command -v g++) -ldl
echo built lidarslam_ros2_b200/csrc/libb200reg.so
# measurement plumbing of bench.py (NVML clock sampling in a native thread), not part of the engine
cd ../../tools
if [ ! -f libclocksampler.so ] || [ clock_sampler.c -nt libclocksampler.so ]; then
  gcc -O2 -shared -fPIC -o libclocksampler.so clock_sampler.c -ldl -lpthread
fi
