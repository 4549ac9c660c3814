"""Top warp-stall sites (SASS level) of every kernel in an .ncu-rep captured with --set full --import-source on:
   python scripts/ncu_hot_sass.py r2_ncu_top.ncu-rep > hot_sass.txt
Reads `ncu -i REP --page source --csv` on the GPU-less host."""
import csv
import io
import re
import subprocess
import sys

rep = sys.argv[1]
top = int(sys.argv[2]) if len(sys.argv) > 2 else 8
out = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"], stdout=subprocess.PIPE, text=True).stdout
blocks = re.split(r'(?m)^"Kernel Name",', out)
seen = set()
print("# {}: top {} warp-stall sampling sites per kernel instantiation (first launch of each)".format(rep, top))
for b in blocks[1:]:
    lines = b.splitlines()
    name = lines[0].strip().strip('",')
    short = re.sub(r"\(CUtensorMap.*", "", name).replace("void b200::", "").replace("b200::", "")
    if short in seen:
        continue
    seen.add(short)
    rows = list(csv.reader(io.StringIO("\n".join(lines[1:]))))
    if not rows:
        continue
    hdr = rows[0]
    try:
        i_src, i_all, i_exec = hdr.index("Source"), hdr.index("Warp Stall Sampling (All Samples)"), hdr.index("Instructions Executed")
    except ValueError:
        continue
    data = []
    for k, r in enumerate(rows[1:]):
        if len(r) <= i_all:
            continue
        try:
            data.append((int(r[i_all]), k, r[i_src].strip(), r[i_exec]))
        except ValueError:
            pass
    total = sum(d[0] for d in data) or 1
    print("\n== {}   ({} SASS instructions, {} stall samples)".format(short[:110], len(data), total))
    for s, k, src, ex in sorted(data, reverse=True)[:top]:
        print("  {:5.1f} %  samples {:6d}  instr #{:<5d} executed {:>8s}   {}".format(100.0 * s / total, s, k, ex, src[:90]))
