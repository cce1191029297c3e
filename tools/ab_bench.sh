#!/bin/bash
# A/B timing of kernel builds: runs `python bench.py ARGS` once per library per round, alternating the libraries, and prints each
# run's JSON line prefixed by the library's name.  Alternation spreads clock and neighbour drift over every build alike.
#   tools/ab_bench.sh ROUNDS "LIB_A LIB_B ..." [bench.py args...]
# A library named "default" is the in-tree build (cpi_b200/libcpi_b200.so).
set -e
cd "$(dirname "$0")/.."
rounds=$1; libs=$2; shift 2
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv,noheader || true
for r in $(seq 1 "$rounds"); do
  for lib in $libs; do
    if [ "$lib" = default ]; then line=$(python bench.py "$@" | tail -1)
    else line=$(CPI_B200_LIB="$lib" python bench.py "$@" | tail -1); fi
    echo "$(basename "$lib") $line"
  done
done
