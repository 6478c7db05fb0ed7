"""Summarise `ncu --set full` reports (read here, no GPU needed) into JSON:
   python tools/ncu_summary.py REPORT.ncu-rep [...] > summary.json
and a launch list (`--metrics gpu__time_duration.sum --csv`) into per-kernel shares:
   python tools/ncu_summary.py --launches LAUNCHES.csv"""
import collections
import csv
import json
import re
import subprocess
import sys

METRICS = {"gpu__time_duration.sum": "gpu_time", "dram__bytes_read.sum": "dram_bytes_read", "dram__bytes_write.sum": "dram_bytes_write",
           "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed": "dram_throughput_pct",
           "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active": "xu_pipe_pct",
           "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active": "tensor_pipe_pct",
           "sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_active": "tensor_hmma_pct",
           "sm__inst_issued.avg.pct_of_peak_sustained_active": "issue_active_pct",
           "sm__warps_active.avg.pct_of_peak_sustained_active": "warps_active_pct",
           "launch__registers_per_thread": "registers_per_thread", "launch__grid_size": "grid", "launch__block_size": "block",
           "sm__throughput.avg.pct_of_peak_sustained_elapsed": "sm_throughput_pct",
           "lts__t_sector_hit_rate.pct": "l2_hit_pct"}


def to_num(v):
    try:
        return float(v.replace(",", ""))
    except ValueError:
        return v


def summarise(rep):
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    if len(rows) < 3:
        return {"report": rep, "error": "unreadable"}
    hdr, units, data = rows[0], rows[1], rows[2]
    out = {"report": rep, "kernel": data[hdr.index("Kernel Name")][:160] if "Kernel Name" in hdr else "?"}
    for i, h in enumerate(hdr):
        if h in METRICS:
            out[METRICS[h]] = to_num(data[i])
            out[METRICS[h] + "_unit"] = units[i]
    if "dram_bytes_read" in out:
        scale = {"Gbyte": 1e9, "Mbyte": 1e6, "Kbyte": 1e3, "byte": 1.0}
        r = out["dram_bytes_read"] * scale.get(out.get("dram_bytes_read_unit", "byte"), 1.0)
        w = out["dram_bytes_write"] * scale.get(out.get("dram_bytes_write_unit", "byte"), 1.0)
        out["traffic_bytes"] = r + w
    return out


def launches(path):
    agg = collections.OrderedDict()
    total = 0.0
    n = 0
    with open(path) as f:
        lines = [ln for ln in f if not ln.startswith("==")]
    for row in csv.DictReader(lines):
        if row.get("Metric Name") != "gpu__time_duration.sum":
            continue
        name = re.sub(r"<.*", "", row["Kernel Name"]).replace("hb::", "").replace("void ", "")
        v = float(row["Metric Value"].replace(",", ""))
        unit = row.get("Metric Unit", "ns")
        ms = v * {"ns": 1e-6, "us": 1e-3, "ms": 1.0, "s": 1e3}.get(unit, 1e-6)
        a = agg.setdefault(name, [0.0, 0])
        a[0] += ms
        a[1] += 1
        total += ms
        n += 1
    print(f"{n} launches, {total:.2f} ms summed (cold-cache, serialised: compare shares)")
    for k, (ms, c) in sorted(agg.items(), key=lambda kv: -kv[1][0]):
        print(f"  {k:34s} {ms:9.3f} ms  {100 * ms / total:5.1f}%  x{c}")


if __name__ == "__main__":
    if sys.argv[1] == "--launches":
        launches(sys.argv[2])
    else:
        print(json.dumps([summarise(r) for r in sys.argv[1:]], indent=1))
