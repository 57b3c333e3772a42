"""Digest of an `ncu --page source --csv` export (gzip) of one kernel: opcode mix by executed instructions and by warp-stall
samples, the stall reasons summed over the kernel, and the SASS lines where warps wait longest.
    ncu --set full --import-source on --clock-control none -k regex:"^msm_accumulate$" -s 1 -c 1 -o acc python tools/profile_workload.py 22 g1
    ncu -i acc.ncu-rep --page source --csv | gzip -9 > ncu_source_accumulate.csv.gz
    python tools/ncu_source_digest.py ncu_source_accumulate.csv.gz "<workload>" "<reading>" > ncu_source_accumulate.md"""
import collections
import csv
import gzip
import io
import re
import sys

rows = list(csv.reader(io.StringIO(gzip.open(sys.argv[1], "rt").read())))
kernel = rows[0][1]
H, data = rows[1], rows[2:]
ix = {h: i for i, h in enumerate(H)}


def f(r, k):
    try:
        return float(r[ix[k]].replace(",", ""))
    except (ValueError, KeyError):
        return 0.0


def opcode(src):
    m = re.match(r"\s*(@!?U?P\d+\s+)?([A-Z0-9_.]+)", src)
    o = m.group(2) if m else "?"
    for pat, name in ((r"^IMAD\.WIDE\S*", "IMAD.WIDE*"), (r"^IMAD\.MOV\S*", "IMAD.MOV"), (r"^IADD3\S*", "IADD3"), (r"^LDG\S*", "LDG"), (r"^STG\S*", "STG"), (r"^LOP3\S*", "LOP3"), (r"^SHF\S*", "SHF"), (r"^ISETP\S*", "ISETP")):
        o = re.sub(pat, name, o)
    return o


tot_i = sum(f(r, "Instructions Executed") for r in data)
tot_s = sum(f(r, "# Samples") for r in data)
tot_n = sum(f(r, "Warp Stall Sampling (Not-issued Samples)") for r in data)
ex, sa, ni = collections.Counter(), collections.Counter(), collections.Counter()
for r in data:
    o = opcode(r[ix["Source"]])
    ex[o] += f(r, "Instructions Executed"); sa[o] += f(r, "# Samples"); ni[o] += f(r, "Warp Stall Sampling (Not-issued Samples)")
print(f"# ncu source page of `{kernel.split('(const')[0].replace('void ', '').replace('b200zk::', '')}` ({sys.argv[2] if len(sys.argv) > 2 else 'workload not stated'}; `tools/ncu_source_digest.py`)\n")
print(f"{len(data)} SASS lines, {tot_i:.3e} warp instructions executed, {int(tot_s)} warp-state samples of which {int(tot_n)} ({100 * tot_n / tot_s:.1f} %) fell in cycles where the")
print("scheduler issued nothing. The full per-line table (stall reasons, L2 sectors, divergence) is the `.csv.gz` next to this file.\n")
print("| opcode | share of executed instructions | share of all samples | share of not-issued samples |")
print("|---|---|---|---|")
for o, v in ex.most_common(10):
    print(f"| `{o}` | {100 * v / tot_i:.1f} % | {100 * sa[o] / tot_s:.1f} % | {100 * ni[o] / tot_n:.1f} % |")
reasons = [h for h in H if h.startswith("stall_") and not h.endswith("(Not Issued)")]
tot_r = {h: sum(f(r, h) for r in data) for h in reasons}
allr = sum(tot_r.values())
print("\n| warp state (all samples) | share |")
print("|---|---|")
for h, v in sorted(tot_r.items(), key=lambda kv: -kv[1])[:9]:
    print(f"| `{h}` | {100 * v / allr:.1f} % |")
print("\n| SASS line (offset) | instruction | samples | not-issued samples | times executed |")
print("|---|---|---|---|---|")
for r in sorted(data, key=lambda r: -f(r, "Warp Stall Sampling (Not-issued Samples)"))[:10]:
    print(f"| `{r[ix['Address']][-5:]}` | `{r[ix['Source']].strip()[:64]}` | {int(f(r, '# Samples'))} | {int(f(r, 'Warp Stall Sampling (Not-issued Samples)'))} | {int(f(r, 'Instructions Executed'))} |")
if len(sys.argv) > 3:
    print("\nReading: " + sys.argv[3])
