#!/bin/bash
# Same-box sweep of library variants (built by tools/build_variants.sh): every variant once per round, rounds interleaved, so that the
# spread between rounds is visible next to the differences between variants. One line per run from tools/probe_variant.py.
#   tools/sweep_variants.sh ROUNDS OUT name[:G] ...    (name -> build/variants/lib_<name>.so; G = lanes per point, default 0)
set -e
cd "$(dirname "$0")/.."
rounds=$1; out=$2; shift 2
mkdir -p "$(dirname "$out")"
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm,clocks.sm,temperature.gpu --format=csv | tee -a "$out"
for r in $(seq 1 "$rounds"); do
  for spec in "$@"; do
    name="${spec%%:*}"; grp=0
    [ "$name" != "$spec" ] && grp="${spec#*:}"
    echo -n "round $r " | tee -a "$out"
    LIINIT_GPU_LIB="build/variants/lib_$name.so" python tools/probe_variant.py "$grp" 2>&1 | tee -a "$out"
  done
done
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm,clocks.sm,temperature.gpu --format=csv | tee -a "$out"
