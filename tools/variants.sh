#!/bin/bash
# Kernel experiments: build single-layout variants of libvsr_b200.so (seconds each) so ONE GPU job can A/B them.
#   tools/variants.sh                       builds build/variants/libvsr_b200_<name>.so for the variants below (cfg2 layout)
#   tools/variants.sh R V K                 same for another layout
# On the GPU machine:  bash tools/ab.sh          (complete BFS of cfg2 with each variant library, three runs each)
# Each variant is the default kernel plus -D flags; "base" has none.
set -e
R=${1:-3}; V=${2:-2}; K=${3:-3}
cd "$(dirname "$0")/../vsr-tlaplus_b200/csrc"
OUT=../../build/variants; mkdir -p $OUT; rm -f $OUT/*.so
ARCH="-gencode arch=compute_90a,code=sm_90a"
ONLY="-DVSR_ONLY_R=$R -DVSR_ONLY_V=$V -DVSR_ONLY_K=$K"
g++ -O2 -std=c++17 -fPIC -c vsr_group.cpp -o $OUT/vsr_group.o
build() { # name, flags
    g++ -O2 -std=c++17 -fPIC $ONLY $2 -c vsr_host.cpp -o $OUT/vsr_host_$1.o   # the host side shares the flags (fingerprints must agree)
    nvcc $ARCH -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -diag-suppress 128 $ONLY $2 -c vsr_gpu.cu -o $OUT/vsr_gpu_$1.o &
    nvcc $ARCH -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -diag-suppress 128 $ONLY $2 -c vsr_shard.cu -o $OUT/vsr_shard_$1.o &
    nvcc $ARCH -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -diag-suppress 128 $ONLY $2 -c vsr_ckpt.cu -o $OUT/vsr_ckpt_$1.o &
    wait
    nvcc $ARCH -shared -Xlinker -Bsymbolic -o $OUT/libvsr_b200_$1.so $OUT/vsr_gpu_$1.o $OUT/vsr_shard_$1.o $OUT/vsr_ckpt_$1.o $OUT/vsr_group.o $OUT/vsr_host_$1.o -ldl -lpthread -lrt
    rm -f $OUT/vsr_gpu_$1.o $OUT/vsr_shard_$1.o $OUT/vsr_ckpt_$1.o $OUT/vsr_host_$1.o
    echo "built $OUT/libvsr_b200_$1.so"
}
build base ""                            # the default: one block of up to 32 warps per SM, pool fast path
build warps16 "-DVSR_FORCE_WARPS=16"     # two blocks of 16 warps per SM (the shape until the re-entry session's A/B: +13 % kernel time)
build nopushfast "-DVSR_EXP_NO_PUSHFAST" # pool layout with the per-pair bound test always (+0.8 %)
build roundclk "-DVSR_EXP_ROUNDCLK"      # per-level split of the expand warps' cycles (end-of-round barrier, scan barriers, batches, scan) on stderr
build passes1 "-DVSR_ROUND_PASSES=1"     # one scan pass per round (the shape before profiles/round_tail_h100.md)
if [ -n "$VSR_VARIANTS_ALL" ]; then
build bucket1 "-DVSR_BUCKET=1"           # seen-set probe = one 128-bit load of one entry (round 1); default is the 2-entry sector bucket
build bucket4 "-DVSR_BUCKET=4"           # 4-entry bucket, two 256-bit loads issued together
fi

build qps1 "-DVSR_QPS=1"                 # correctness variant (pool overflow path): VSR_B200_LIB=...qps1.so python -m pytest tests/test_gpu_parity.py -k "3-2-2 or deterministic"
build weakfp "-DVSR_WEAK_FP_BITS=16"     # correctness variant (16-bit fingerprints: collisions everywhere, kept apart by the check hash; tests/test_fp_collisions.py)
rm -f $OUT/vsr_group.o
