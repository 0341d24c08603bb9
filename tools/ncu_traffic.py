#!/usr/bin/env python3
"""profiles/traffic.json + the headline ncu metrics of the dominant kernel from an ncu --set full report.
Usage: tools/ncu_traffic.py <report.ncu-rep> <out_metrics.json> [<out_traffic.json>]"""
import csv, json, subprocess, sys

rep, out_metrics = sys.argv[1], sys.argv[2]
out_traffic = sys.argv[3] if len(sys.argv) > 3 else "profiles/traffic.json"
rows = list(csv.reader(subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout.splitlines()))
hdr, units, data = rows[0], rows[1], rows[2:]
want = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread", "smsp__inst_executed.sum", "sm__cycles_elapsed.max",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__warps_eligible.avg.per_cycle_active", "lts__t_sector_hit_rate.pct",
        "l1tex__t_sector_hit_rate.pct", "launch__grid_size", "launch__block_size", "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed"]
scale = {"Mbyte": 1e6, "Kbyte": 1e3, "byte": 1.0, "Gbyte": 1e9}
launches = []
for d in data:
    rec = {"kernel": d[hdr.index("Kernel Name")], "device": d[hdr.index("device__attribute_display_name")]}
    for w in want:
        if w in hdr:
            i = hdr.index(w); rec[w] = {"value": d[i], "unit": units[i]}
    launches.append(rec)
json.dump({"source": "ncu --set full --clock-control none, read with ncu -i ... --page raw --csv", "k_bricks": launches}, open(out_metrics, "w"), indent=0)
k = launches[-1]
rd = float(k["dram__bytes_read.sum"]["value"]) * scale[k["dram__bytes_read.sum"]["unit"]]
wr = float(k["dram__bytes_write.sum"]["value"]) * scale[k["dram__bytes_write.sum"]["unit"]]
# bench.py uses the figure only on a device of this name (a capture of one GPU model says nothing about another)
json.dump({"kernel": "k_bricks<COLOR=1, MINB=6>", "device": k["device"], "dram_bytes_per_launch": rd + wr, "dram_read": rd, "dram_write": wr,
           "source": "ncu --set full, one launch of the bench workload at N=1 (frame 20 of tools/prof_integrate.py)"}, open(out_traffic, "w"), indent=1)
print("k_bricks dram bytes/launch", rd + wr, "time", k["gpu__time_duration.sum"])
