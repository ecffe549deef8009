#!/bin/bash
# Time several builds of the kernels in ONE GPU session.
#   here (no GPU):   make -C traversability_estimation_b200/csrc variant NAME=a EXTRA="-DX=1"   (one per variant)
#   under gpurun:    bash tools/dev_variants.sh a b c -- --holes 0
# Every variant is libte_b200_<name>.so next to the product library; "base" means the product library itself.
names=(); extra=()
while [ $# -gt 0 ]; do
  if [ "$1" == "--" ]; then shift; extra=("$@"); break; fi
  names+=("$1"); shift
done
mkdir -p gpurun_out
for n in base "${names[@]}"; do
  lib=""; [ "$n" != "base" ] && lib="$PWD/traversability_estimation_b200/libte_b200_$n.so"
  TE_B200_LIBRARY="$lib" timeout 300 python bench.py --steps 20 --warmup 3 --no-cpu-baseline --no-e2e "${extra[@]}" 2>> gpurun_out/err_variants.log | python -c "
import json,sys; d=json.loads(sys.stdin.read()); print('$n', round(d['value']), d['ms_per_step'], d['roofline'].get('kernel_ms'), d['roofline'].get('fixup_kernel_ms'))"
done
tail -3 gpurun_out/err_variants.log
