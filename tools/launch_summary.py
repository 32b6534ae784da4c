"""Per-kernel totals of an `ncu --metrics gpu__time_duration.sum --csv` launch list.

    python tools/launch_summary.py launches.csv
"""
import csv
import re
import sys
from collections import defaultdict

rows = [r for r in csv.reader(open(sys.argv[1])) if len(r) > 14 and r[0].isdigit()]
tot, cnt = defaultdict(float), defaultdict(int)
for r in rows:
    name = re.sub(r"\(.*", "", r[4]).replace("void ", "").replace("b200rl::", "")
    tot[name] += float(r[14].replace(",", "")) / 1e3
    cnt[name] += 1
total = sum(tot.values())
print(f"{len(rows)} launches, {total / 1e3:.2f} ms of kernel time")
for k in sorted(tot, key=lambda k: -tot[k]):
    print(f"| `{k}` | {cnt[k]} | {tot[k] / 1e3:.2f} ms | {tot[k] / cnt[k]:.1f} us | {100 * tot[k] / total:.1f} % |")
