"""Formats `nvcc -Xptxas -v` logs (one per translation unit) as a markdown table; see ptxas_table.sh."""
import glob
import re
import subprocess
import sys

rows = []
for p in sorted(glob.glob(sys.argv[1] + "/*.log")):
    name, st = None, ("0", "0", "0")
    for line in open(p):
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            name = m.group(1)
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            st = m.groups()
        m = re.search(r"Used (\d+) registers(?:, used (\d+) barriers)?(?:, (\d+) bytes smem)?", line)
        if m and name:
            dem = subprocess.run(["c++filt", name], capture_output=True, text=True).stdout.strip()
            dem = re.sub(r"\(.*", "", dem).replace("mvs::", "")
            rows.append((p.split("/")[-1][:-4] + ".cu", dem, m.group(1), m.group(3) or "0", *st))
            name = None
print("# ptxas resource table, sm_90a (`scripts/ptxas_table.sh`; static shared memory only — the resident,")
print("# frame_step, sdf_fused, skin and GEMM kernels take their shared memory dynamically, see DESIGN.md §4)\n")
print("| file | kernel | registers | static smem B | stack B | spill st/ld B |")
print("|---|---|---:|---:|---:|---:|")
for r in rows:
    print(f"| {r[0]} | `{r[1]}` | {r[2]} | {r[3]} | {r[4]} | {r[5]}/{r[6]} |")
