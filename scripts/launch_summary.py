#!/usr/bin/env python
"""ncu launch list (--metrics gpu__time_duration.sum --csv) -> markdown table.
    python scripts/launch_summary.py launches.csv "title" [n_steps_in_list] > launch_summary.md
Per-launch times under ncu are cold-cache and serialised: compare SHARES, not absolutes."""
import collections
import csv
import sys

path, title = sys.argv[1], sys.argv[2]
steps = float(sys.argv[3]) if len(sys.argv) > 3 else None
with open(path) as f:
    lines = [l for l in f if not l.startswith("==")]
agg = collections.OrderedDict()
for row in csv.DictReader(lines):
    if row.get("Metric Name") != "gpu__time_duration.sum":
        continue
    v = float(row["Metric Value"])
    if row["Metric Unit"] == "ns":
        v /= 1e3
    elif row["Metric Unit"] == "ms":
        v *= 1e3
    k = row["Kernel Name"]
    a = agg.setdefault(k, [0, 0.0])
    a[0] += 1
    a[1] += v
tot = sum(v[1] for v in agg.values())
n = sum(v[0] for v in agg.values())
print("# %s\n" % title)
print("Per-launch times under ncu are cold-cache and serialised: compare SHARES, not absolutes.\n")
print("| kernel | launches | avg us | total us | share |\n|---|---|---|---|---|")
for k, (c, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
    print("| `%s` | %d | %.1f | %.1f | %.1f%% |" % (k[:90], c, t / c, t, 100 * t / tot))
print("\nTotal %.0f us over %d launches%s." % (tot, n, (" = %.1f launches and %.0f us per step" % (n / steps, tot / steps)) if steps else ""))
