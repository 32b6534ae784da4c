"""Summarise one `ncu --set full` capture into the small JSON bench.py quotes (dram bytes per launch, issue / tensor
pipe utilisation) and a CSV of the raw page.

    python tools/ncu_summary.py report.ncu-rep summary.json [raw.csv]
"""
import csv
import io
import json
import subprocess
import sys

rep, out = sys.argv[1], sys.argv[2]
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
h, u, v = rows[0], rows[1], rows[2]
m = {n: (v[i], u[i]) for i, n in enumerate(h)}


def f(name):
    return float(m[name][0].replace(",", ""))


def bytes_of(name):
    val, unit = f(name), m[name][1].lower()
    return val * {"byte": 1, "kbyte": 1e3, "mbyte": 1e6, "gbyte": 1e9}[unit]


summary = {
    "source": rep.split("/")[-1] + " (ncu --set full --clock-control none)",
    "kernel": m["Kernel Name"][0],
    "duration_us": f("gpu__time_duration.sum"),
    "dram_read_bytes": bytes_of("dram__bytes_read.sum"),
    "dram_write_bytes": bytes_of("dram__bytes_write.sum"),
    "dram_bytes_per_launch": bytes_of("dram__bytes_read.sum") + bytes_of("dram__bytes_write.sum"),
    "warp_instructions": f("smsp__inst_executed.sum"),
    "issue_active_pct": f("smsp__issue_active.avg.pct_of_peak_sustained_active"),
    "tensor_pipe_active_pct": f("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active"),
    "registers": f("launch__registers_per_thread"),
    "stalls_per_issue": {k.split("issue_stalled_")[1].split("_per_issue")[0]: float(val[0])
                         for k, val in m.items() if k.startswith("smsp__average_warps_issue_stalled") and "per_issue_active" in k},
}
json.dump(summary, open(out, "w"), indent=1)
print(json.dumps(summary, indent=1))
if len(sys.argv) > 3:
    keep = [i for i, n in enumerate(h) if any(t in n for t in ("Kernel Name", "gpu__time", "dram__bytes", "smsp__inst_executed.sum",
            "smsp__issue_active", "sm__pipe_tensor_cycles_active", "issue_stalled", "launch__registers", "sm__throughput",
            "sm__inst_executed_pipe", "l1tex__data_bank", "lts__t_sector_hit"))]
    with open(sys.argv[3], "w", newline="") as fo:
        w = csv.writer(fo)
        for i in keep:
            w.writerow([h[i], u[i], v[i]])
