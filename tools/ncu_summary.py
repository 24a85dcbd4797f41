"""Summarise an .ncu-rep (read here, without a GPU) into a small text file."""
import csv
import subprocess
import sys

KEYS = ["gpu__time_duration.sum", "sm__cycles_active.avg", "sm__cycles_elapsed.avg.per_second",
        "sm__pipe_tensor_cycles_active_realtime.avg.pct_of_peak_sustained_elapsed",
        "sm__inst_executed_pipe_tensor.sum", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "derived__lts__lts2xbar_bytes.sum.per_second", "lts__t_sectors.sum", "lts__t_sector_hit_rate.pct",
        "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "smsp__inst_executed.sum",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "launch__registers_per_thread", "launch__grid_size", "launch__block_size", "launch__cluster_size",
        "launch__shared_mem_per_block_dynamic"]


def main(rep, out):
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    hdr, units = rows[0], rows[1]
    idx = {h: i for i, h in enumerate(hdr)}
    with open(out, "w") as f:
        f.write(f"# ncu --set full --clock-control none summary of {rep}\n")
        for n, r in enumerate(rows[2:]):
            f.write(f"\n## launch {n}: {r[idx['Kernel Name']][:160]}\n")
            for k in KEYS:
                hit = [h for h in hdr if h == k or h.endswith("." + k) or h.endswith(k)]
                if hit:
                    h = hit[0]
                    f.write(f"{k:85s} {r[idx[h]]:>18s} {units[idx[h]]}\n")
            tr = float(r[idx["dram__bytes_read.sum"]] or 0) + float(r[idx["dram__bytes_write.sum"]] or 0)
            f.write(f"{'traffic = dram__bytes_read.sum + dram__bytes_write.sum':85s} {tr:18.3f} {units[idx['dram__bytes_read.sum']]}\n")
    src = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(src.splitlines()))
    if len(rows) > 2:
        hdr = rows[1]
        si, k = hdr.index("Source"), hdr.index("# Samples")
        body = []
        for r in rows[2:]:
            if len(r) > k and r[k].replace(".", "").isdigit():
                body.append(r)
            elif body and r and r[0] == "Kernel Name":
                break  # next launch
        tot = sum(float(r[k]) for r in body) or 1.0
        with open(out, "a") as f:
            f.write("\n## hottest SASS instructions of the first launch (share of warp-state samples)\n")
            for r in sorted(body, key=lambda r: -float(r[k]))[:15]:
                f.write(f"{float(r[k]) / tot * 100:6.2f}%  {r[si].strip()[:120]}\n")


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
