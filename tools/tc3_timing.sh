#!/bin/bash
# A/B build of the fused PPO step with its per-tile cycle counters (run from the repo root after build.py):
#   tools/tc3_timing.sh     -> tools/bin/libb200rl_tc3_timing.so
#   B200RL_TC3_TIMING=1 B200RL_LIB=tools/bin/libb200rl_tc3_timing.so python tools/profile_fused.py
# The counters live in a 512-byte local array, so the timing build runs slower than the library: read its cycle counts
# as shares of a tile, not as absolute times.
set -e
PK=reinforcement-learning-replications_b200
FL="-O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -Xcompiler -fPIC -Xcompiler -fvisibility=default -I include -I $PK/csrc"
mkdir -p tools/bin
others=$(ls $PK/build/*.o | grep -v mlp_tc3)
nvcc $FL -DB200RL_TC3_TIMING -c -o tools/bin/mlp_tc3_timing.o $PK/csrc/mlp_tc3.cu
nvcc --shared -cudart static -gencode arch=compute_90a,code=sm_90a -o tools/bin/libb200rl_tc3_timing.so tools/bin/mlp_tc3_timing.o $others
