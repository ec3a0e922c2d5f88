"""Text summary of an ncu report (read on the CPU box): per profiled launch the duration, DRAM
bytes, pipe utilisations, occupancy limits and the top warp-stall reasons.

    python tools/ncu_summary.py kernels.ncu-rep > kernels_summary.txt
"""
import csv
import io
import subprocess
import sys

KEYS = [
    "launch__grid_size", "launch__block_size", "gpu__time_duration.sum",
    "dram__bytes_read.sum", "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "smsp__issue_active.avg.pct_of_peak_sustained_active",
    "sm__warps_active.avg.pct_of_peak_sustained_active",
    "launch__registers_per_thread", "launch__shared_mem_per_block_dynamic",
    "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem",
    "sm__cycles_elapsed.avg.per_second", "lts__t_sector_hit_rate.pct",
    "l1tex__t_sector_hit_rate.pct",
]


def page(rep, name):
    out = subprocess.run(["ncu", "-i", rep, "--page", name, "--csv"], capture_output=True,
                         text=True).stdout
    return list(csv.reader(io.StringIO(out)))


def main():
    rep = sys.argv[1]
    rows = page(rep, "raw")
    hdr, units = rows[0], rows[1]
    print("ncu -i %s  (--set full --clock-control none; durations under ncu are cold-cache, "
          "serialised and at unlocked clocks: not bench values)\n" % rep)
    src = page(rep, "source")
    # the source page lists every profiled launch in order (SASS view, then the source view of
    # the same launch): keep the first table of each launch
    tables, st = [], None
    for r in src:
        if r and r[0] == "Kernel Name":
            st = {"name": r[1], "hdr": None, "agg": {}}
            tables.append(st)
            continue
        if st is None or not r:
            continue
        if r[0] == "Address" or st["hdr"] is None:
            st["hdr"] = r
            st["cols"] = [i for i, h in enumerate(r)
                          if h.startswith("stall_") and "Not Issued" not in h]
            continue
        for i in st["cols"]:
            try:
                st["agg"][st["hdr"][i]] = st["agg"].get(st["hdr"][i], 0) + int(r[i] or 0)
            except (ValueError, IndexError):
                pass
    per_launch = []
    for t in tables:
        if per_launch and per_launch[-1]["name"] == t["name"] and len(per_launch) * 2 > len(tables):
            continue
        per_launch.append(t)
    if len(tables) == 2 * (len(rows) - 2):
        per_launch = tables[::2]
    for r in rows[2:]:
        name = r[hdr.index("Kernel Name")]
        print("=== " + name)
        for k in KEYS:
            if k in hdr:
                i = hdr.index(k)
                print("    %-66s %s %s" % (k, r[i], units[i]))
        k = rows.index(r) - 2
        if k < len(per_launch) and per_launch[k]["agg"]:
            agg = per_launch[k]["agg"]
            tot = sum(agg.values()) or 1
            top = sorted(agg.items(), key=lambda kv: -kv[1])[:6]
            print("    warp stall samples (all warps incl. idle / waiting roles): " +
                  ", ".join("%s %.0f%%" % (n.replace("stall_", ""), 100.0 * v / tot)
                            for n, v in top))
        print()


if __name__ == "__main__":
    main()
