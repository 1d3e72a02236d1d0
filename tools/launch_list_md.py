"""tools/launch_list_md.py -- turn an `ncu --metrics gpu__time_duration.sum --csv` launch list into the per-kernel
share table in markdown.   usage: python tools/launch_list_md.py launches.csv out.md "<title line>" """
import csv
import re
import sys
from collections import defaultdict

src, dst, title = sys.argv[1], sys.argv[2], sys.argv[3]
rows = [ln for ln in open(src, newline="") if ln.startswith('"')]
tot, cnt = defaultdict(float), defaultdict(int)
for r in csv.DictReader(rows):
    if r["Metric Name"] != "gpu__time_duration.sum":
        continue
    name = re.sub(r"\(.*", "", r["Kernel Name"]).replace("void ", "").strip()
    name = name.split("::")[-1]
    tot[name] += float(r["Metric Value"]) / 1e6
    cnt[name] += 1
allms = sum(tot.values())
with open(dst, "w") as f:
    f.write(f"# {title}\n\n(cold-cache, serialised per-launch times: compare shares, not absolutes)\n\n")
    f.write("| kernel | launches | total ms | share |\n|---|---|---|---|\n")
    for k in sorted(tot, key=tot.get, reverse=True):
        f.write(f"| `{k}` | {cnt[k]} | {tot[k]:.3f} | {tot[k] / allms:.4f} |\n")
print(open(dst).read())
