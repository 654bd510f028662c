#!/bin/bash
# GPU side of tools/variants.sh: complete BFS of cfg2 with each variant library, three runs each, kernel seconds and rates.
# usage (on the GPU machine):  bash tools/ab.sh [R V L]      (default 3 2 2 = shipped VSR.cfg)
R=${1:-3}; V=${2:-2}; L=${3:-2}; TABLE=${4:-0}; FRONTIER=${5:-0}
for v in build/variants/libvsr_b200_*.so; do
    for i in 1 2 3; do
        QUIET=1 VSR_B200_LIB=$v python tools/quick.py $R $V $L 0 0 $TABLE $FRONTIER | head -1 | python -c "
import json, sys
d = json.loads(sys.stdin.readline())
print('%-46s kern %.4f s  total %.4f s  %.3e distinct/s (kernel)  probes/gen %.3f  distinct %d' % ('$v'.split('/')[-1], d['kern'], d['secs'], d['krate'], d['probes_per_gen'], d['distinct']))"
    done
done
