#!/bin/bash
# usage: tools/conv_decomp.sh <tag> "<dbg masks>" [lib ...] — bench.py per lib (default: the product lib) with parts of the conv
# kernel switched off (B200AD_CONV_DBG: 2 = no global stores, 8 = no epilogue work, 32 = no weight loads,
# 64 = no transform); prints conv_tc ms per step.
tag=$1; masks=$2; shift 2
libs=${@:-audio_diffusion_b200/libb200ad.so}
for lib in $libs; do
  for d in $masks; do
    B200AD_LIB=$PWD/$lib B200AD_CONV_DBG=$d timeout 300 python bench.py --steps 5 --warmup 3 --no-cpu --no-extras 2>/dev/null | python -c "
import sys, json
d = json.loads(sys.stdin.read())
print('$lib', 'dbg', $d, 'conv_tc ms', d['roofline']['ms_by_kernel']['conv_tc'], 'step ms', round(d['ms_per_step'], 2))" | tee -a gpurun_out/conv_decomp_$tag.txt
  done
done
