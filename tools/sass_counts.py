"""Mnemonic counts per kernel of libb200rl.so.

    python tools/sass_counts.py [path/to/libb200rl.so]
"""
import re
import subprocess
import sys

lib = sys.argv[1] if len(sys.argv) > 1 else "reinforcement-learning-replications_b200/libb200rl.so"
sass = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
cols = ["UTCHMMA", "LDTM", "STTM", "UTCBAR", "UBLKCP", "SYNCS", "LDGSTS", "MUFU"]
want = re.compile(r"gae_scan|mlp_tc|tc_probe|reduce_adam3")
print("| kernel | instructions | " + " | ".join(cols) + " |")
print("|---|" + "---|" * (len(cols) + 1))
for block in sass.split("Function : ")[1:]:
    name = block.split("\n", 1)[0].strip()
    if not want.search(name):
        continue
    ins = re.findall(r"^\s*/\*[0-9a-f]{4,6}\*/\s+(?:@!?U?P\d\s+)?([A-Z0-9_.]+)", block, flags=re.M)
    counts = [sum(1 for i in ins if i.split(".")[0] == c) for c in cols]
    print(f"| `{name}` | {len(ins)} | " + " | ".join(str(c) for c in counts) + " |")
