#!/bin/bash
# Static resource table (registers / stack / spills / static smem) of every kernel, cross-compiled for sm_90a.
# No GPU needed.  Output: markdown on stdout
set -e
cd "$(dirname "$0")/.."
T=$(mktemp -d)
for f in mvsmplfitting_b200/csrc/*.cu; do
  b=$(basename "$f" .cu)
  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Iinclude -Xptxas -v -c "$f" -o "$T/$b.o" 2> "$T/$b.log"
done
python scripts/ptxas_table.py "$T"
rm -rf "$T"
