"""Summarise `ncu --metrics gpu__time_duration.sum --csv` output into shares per kernel."""
import csv
import re
import sys
from collections import defaultdict


def main(path, out, header):
    rows = []
    with open(path, newline="") as f:
        lines = [ln for ln in f if ln.startswith('"')]
    rd = csv.reader(lines)
    hdr = next(rd)
    ki, mi, vi, ui = hdr.index("Kernel Name"), hdr.index("Metric Name"), hdr.index("Metric Value"), hdr.index("Metric Unit")
    agg = defaultdict(lambda: [0, 0.0])
    for r in rd:
        if len(r) <= vi or r[mi] != "gpu__time_duration.sum":
            continue
        v = float(r[vi].replace(",", ""))
        us = v / 1e3 if r[ui] in ("ns", "nsecond") else v * 1e3 if r[ui] in ("ms", "msecond") else v
        name = re.sub(r"\(.*$", "", r[ki]).strip()
        agg[name][0] += 1
        agg[name][1] += us
    tot = sum(v[1] for v in agg.values()) or 1.0
    with open(out, "w") as f:
        f.write(header.rstrip() + "\n")
        f.write(f"# total launches {sum(v[0] for v in agg.values())}, total kernel time {tot / 1e3:.1f} ms\n")
        f.write("  share  launches     total_us    avg_us  kernel\n")
        for name, (n, us) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            f.write(f"{us / tot * 100:6.2f}%  {n:8d}  {us:11.1f}  {us / n:8.2f}  {name[:150]}\n")


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2], sys.argv[3] if len(sys.argv) > 3 else "# ncu launch list")
