#!/bin/bash
# Tuning sweep of the fast chain's launch choices on the C3 frame at 4K (run on the GPU after build()); one line per setting.
#   run time:     RFX_K3_TMA (TMA-staged tap tiles of the Poisson passes >= 1)
#   compile time: RFX_K1_BATCH (K1 march steps fetched together), RFX_K1_MIN_BLOCKS (K1's __launch_bounds__ minimum resident
#                 blocks per SM); only k_ssgi.cu is rebuilt
# Leaves the default build in place.
cd "$(dirname "$0")/.."
time_line() {  # label, then environment assignments for bench.py
  label=$1; shift
  env "$@" python bench.py --steps 50 --warmup 5 --no-cpu-baseline --no-configs 2>/dev/null | tail -1 | python -c "
import json, sys
d = json.loads(sys.stdin.read()); pk = d['roofline']['per_kernel']
print('$label | frame ms', d['ms_per_step'], '| K1 ms', round(pk['K1_ssgi_trace']['ms_per_launch'], 3),
      '| K3 pass>=1 ms', round(pk['K3_poisson_pass1plus']['ms_per_launch'], 3), '|', d['device'])"
}
rebuild_k1() {  # extra nvcc flags for k_ssgi.cu
  rm -f realism_effects_b200/csrc/build/k_ssgi.o
  RFX_NVCC_EXTRA="$1" python -c "import __graft_entry__ as g; g.build()" > /dev/null 2>&1
}
for t in 0 1; do time_line "RFX_K3_TMA=$t" RFX_K3_TMA=$t; done
for b in 1 2; do
  rebuild_k1 "-DRFX_K1_BATCH=$b"
  time_line "RFX_K1_BATCH=$b"
done
for mb in 3 5 4; do  # 4 (the default, with the default batch) last, so that the default build is what stays
  rebuild_k1 "-DRFX_K1_MIN_BLOCKS=$mb"
  time_line "RFX_K1_MIN_BLOCKS=$mb"
done
