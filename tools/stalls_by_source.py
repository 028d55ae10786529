#!/usr/bin/env python
"""Warp-stall samples of one kernel by CUDA source line, from an ncu report.

  ncu -i X.ncu-rep --page source --csv --print-source sass > src.csv
  cuobjdump -xelf all sortmerna_b200/libsmr_b200.so && nvdisasm -g -c smr_capi.sm_90a.cubin > disasm.txt
  python tools/stalls_by_source.py src.csv disasm.txt '.text._ZN3smr10lis_kernel'

The ncu source page gives samples per SASS address; nvdisasm -g gives the source line of every SASS offset of the same cubin."""
import collections
import csv
import re
import sys


def main(src_csv, disasm, kernel_section, top=40):
    lines = open(disasm).read().split("\n")
    start = next(i for i, l in enumerate(lines) if kernel_section in l)
    end = next((i for i in range(start + 1, len(lines)) if lines[i].startswith("//---") and ".text." in lines[i]), len(lines))
    cur, offmap = None, {}
    for l in lines[start:end]:
        m = re.search(r'//## File "([^"]+)", line (\d+)', l)
        if m:
            cur = (m.group(1).split("/")[-1], int(m.group(2)))
            continue
        m = re.match(r"\s+/\*([0-9a-f]{4,6})\*/", l)
        if m:
            offmap[int(m.group(1), 16)] = cur
    rows = list(csv.reader(open(src_csv)))
    hdr = rows[1]
    data = [r for r in rows[2:] if len(r) >= len(hdr)]
    ix = {h: i for i, h in enumerate(hdr)}
    stalls = [h for h in hdr if h.startswith("stall_") and "Not Issued" not in h]
    base = int(data[0][ix["Address"]], 16)
    tot, T = collections.Counter(), 0
    agg = collections.defaultdict(collections.Counter)
    for r in data:
        n = int(r[ix["# Samples"]] or 0)
        T += n
        key = offmap.get(int(r[ix["Address"]], 16) - base)
        agg[key]["samples"] += n
        for s in stalls:
            v = int(r[ix[s]] or 0)
            tot[s] += v
            agg[key][s] += v
    print(f"{T} samples")
    for s, v in tot.most_common(10):
        print(f"  {s:26s} {100 * v / T:5.1f}%")
    for key, c in sorted(agg.items(), key=lambda x: -x[1]["samples"])[:top]:
        best = sorted(((s, c[s]) for s in stalls), key=lambda x: -x[1])[:2]
        print(key, f"{100 * c['samples'] / T:5.2f}%", [(s[6:], round(100 * v / T, 2)) for s, v in best])


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2], sys.argv[3])
