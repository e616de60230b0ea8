#!/bin/bash
# Build promp_b200/libpromp_b200_clk.so: the same sources with -DPROMP_EXP_CLOCKS (per-phase clock64 counters; experiments only).
set -e
cd "$(dirname "$0")/.."
mkdir -p build/obj_clk
for f in common rollout process policy policy_relu policy_otanh policy_relu_otanh comm trpo paths; do
  nvcc -std=c++17 -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -Xcompiler -fPIC -DPROMP_EXP_CLOCKS -c promp_b200/csrc/$f.cu -o build/obj_clk/$f.o &
done
wait
nvcc -shared -o promp_b200/libpromp_b200_clk.so build/obj_clk/*.o
ls -la promp_b200/libpromp_b200_clk.so
