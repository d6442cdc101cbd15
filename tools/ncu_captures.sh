#!/bin/bash
# `ncu --set full` captures of the tensor-core kernels, one small CSV (raw page) per kernel under
# gpurun_out/ (the .ncu-rep files are deleted on the box: gpurun_out is capped at 64 MiB).   bash tools/ncu_captures.sh <tag>
TAG=${1:-r2}; O=gpurun_out; mkdir -p $O
cap() {  # name, kernel regex, launch-skip, launch-count, extra env
  local name=$1 re=$2 skip=$3 cnt=$4; shift 4
  env "$@" ncu --set full --clock-control none --kernel-name-base demangled -k "regex:$re" --launch-skip $skip --launch-count $cnt \
      -f -o /tmp/ncu_$name python tools/profile_kernels.py > $O/${TAG}_ncu_${name}.out 2>&1
  ncu -i /tmp/ncu_$name.ncu-rep --page raw --csv > $O/${TAG}_ncu_${name}.csv 2>/dev/null
  rm -f /tmp/ncu_$name.ncu-rep
}
# exemplar prologue = 41 tensor-core conv launches; frame kernels come after.  Pick launches of the first frame.
cap conv256 'conv_tc_kernel<\(int\)256' 24 8 DVC_X=1
cap conv128 'conv_tc_kernel<\(int\)128' 14 4 DVC_X=1
cap conv64  'conv_tc_kernel<\(int\)64' 8 3 DVC_X=1
cap xform   'xform_kernel'       20 4 DVC_X=1
cap screen  'corr_screen_kernel' 0 1 DVC_X=1
cap rescore 'corr_rescore_kernel' 0 1 DVC_X=1
cap corr3   'corr_tc_kernel'     0 1 DVC_SCREEN=0
cap softmax 'corr_tc_kernel'     0 1 DVC_T=0.01
ls -la $O | grep ncu
