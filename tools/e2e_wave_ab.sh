#!/bin/bash
# e2e A/B of the host entry's tail handling (run from the repo root)
B="python bench.py --no-cpu-baseline --no-configs --no-clocks --steps 50 --warmup 3"
for spec in "0,0" "14,8" "8,8" "24,8" "14,4" "14,16" "32,8" "0,0" "14,8"; do
  echo "== wave G,S $spec"
  CPI_B200_HOST_WAVE=$spec $B 2>/dev/null | python -c "
import json,sys
d=json.loads(sys.stdin.read().strip().splitlines()[-1]); e=d['e2e']
print('e2e %.3f ms  %.3f M/s   floor h2d %.3f ms (%.1f GB/s)  kernel %.3f' % (e['ms_per_step'], e['value']/1e6, e['pcie_floor']['h2d_ms'], e['pcie_floor']['h2d_gbs'], d['kernel_ms']))"
done
