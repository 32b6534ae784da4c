#!/bin/bash
# A/B builds of the episode scan kernel with other ring / occupancy settings (run from the repo root after build.py):
#   tools/scan_variants.sh            -> tools/bin/libb200rl_<name>.so
#   B200RL_LIB=tools/bin/libb200rl_<name>.so python tools/profile_scan.py
set -e
PK=reinforcement-learning-replications_b200
FL="-O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -Xcompiler -fPIC -Xcompiler -fvisibility=default -I include -I $PK/csrc"
mkdir -p tools/bin
others=$(ls $PK/build/*.o | grep -v gae_scan)
build() {  # name, defines
  nvcc $FL $2 -c -o tools/bin/gae_scan_$1.o $PK/csrc/gae_scan.cu
  nvcc --shared -cudart static -gencode arch=compute_90a,code=sm_90a -o tools/bin/libb200rl_$1.so tools/bin/gae_scan_$1.o $others
  cuobjdump -res-usage tools/bin/libb200rl_$1.so 2>/dev/null | grep -A1 "gae_scan_episode_kernelId" | grep REG | sed "s/^/$1: /"
}
build minb1 "-DB200RL_EP_MINB=1"
build w10s3 "-DB200RL_EP_WARPS=10 -DB200RL_EP_STAGES=3 -DB200RL_EP_CTAS=2 -DB200RL_EP_MINB=2"
build w12s3 "-DB200RL_EP_WARPS=12 -DB200RL_EP_STAGES=3 -DB200RL_EP_CTAS=2 -DB200RL_EP_MINB=2"
