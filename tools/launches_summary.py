"""ncu launch list (`--metrics gpu__time_duration.sum --csv`) -> markdown: per-kernel time and share of the listed launches.
    python tools/launches_summary.py launches_ncu.csv > launches_summary.md"""
import collections
import csv
import sys

rows = list(csv.reader([l for l in open(sys.argv[1]) if not l.startswith("==")]))
hdr = rows[0]
kn, mv, mu = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("Metric Unit")
scale = {"ns": 1e-6, "us": 1e-3, "ms": 1.0, "nsecond": 1e-6, "usecond": 1e-3, "msecond": 1.0}
tot, cnt = collections.OrderedDict(), collections.Counter()
for r in rows[1:]:
    if len(r) != len(hdr):
        continue
    name = r[kn].split("(")[0].replace("b200zk::", "").replace("Fe<FqCfg>", "Fq").replace("void ", "")
    tot[name] = tot.get(name, 0.0) + float(r[mv].replace(",", "")) * scale.get(r[mu], 1.0)
    cnt[name] += 1
total = sum(tot.values())
print("| kernel | launches | time (ms, ncu: cold-cache, serialised) | share |")
print("|---|---|---|---|")
for k, v in sorted(tot.items(), key=lambda kv: -kv[1]):
    print(f"| `{k}` | {cnt[k]} | {v:.3f} | {100 * v / total:.1f} % |")
print(f"| **total** | {sum(cnt.values())} | {total:.3f} | 100 % |")
