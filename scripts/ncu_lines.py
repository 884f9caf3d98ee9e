#!/usr/bin/env python
"""Per-source-line summary of an ncu report (compiled with -lineinfo, captured with --import-source on):
    python scripts/ncu_lines.py prof.ncu-rep [top_n]
prints the share of executed warp instructions and of stall samples per CUDA source line, with the two dominant stall reasons."""
import csv
import io
import subprocess
import sys

rep, top = sys.argv[1], int(sys.argv[2]) if len(sys.argv) > 2 else 40
txt = subprocess.run(["ncu", "-i", rep, "--page", "source", "--print-source", "cuda,sass", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(txt)))
fname, hdr, data = "", None, []
for r in rows:
    if not r:
        continue
    if r[0] == "File Path":
        fname = r[1].split("/")[-1]
    elif r[0] == "Line No":
        hdr = r
    elif hdr and len(r) == len(hdr) and r[2] == "-":          # a source-line aggregate (its SASS rows carry an address instead)
        ix = {n: i for i, n in enumerate(hdr)}
        try:
            inst, samp = int(r[ix["Instructions Executed"]]), int(r[ix["# Samples"]])
        except ValueError:
            continue
        stalls = sorted(((int(r[i] or 0), h[6:]) for i, h in enumerate(hdr) if h.startswith("stall_") and "Not Issued" not in h), reverse=True)[:2]
        data.append((fname, int(r[0]), r[1].strip(), inst, samp, stalls))
ti, ts = sum(d[3] for d in data) or 1, sum(d[4] for d in data) or 1
print(f"warp instructions {ti}, stall samples {ts}")
for f, ln, src, inst, samp, st in sorted(data, key=lambda d: -d[4])[:top]:
    print(f"{f}:{ln:<4d} inst {100 * inst / ti:5.1f}%  samples {100 * samp / ts:5.1f}%  {st[0][1]}:{st[0][0]} {st[1][1]}:{st[1][0]} | {src[:120]}")
