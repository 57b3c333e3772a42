"""A markdown excerpt (on stdout) of the built libb200zk.so: per-kernel SASS mnemonic counts (cuobjdump -sass) and resource
usage (cuobjdump -res-usage) -- the evidence that the shipped kernels are sm_90a code built from IMAD.WIDE carry chains and
bulk-copy (TMA) staging, with no tensor-core or legacy paths.   python tools/sass_excerpt.py > sass_excerpt.md"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "ethrex_b200", "libb200zk.so")
sys.path.insert(0, ROOT)
import bench  # noqa: E402

sass = subprocess.run(["cuobjdump", "-sass", SO], capture_output=True, text=True, check=True).stdout
res = subprocess.run(["cuobjdump", "-res-usage", SO], capture_output=True, text=True, check=True).stdout
demangle = lambda names: dict(zip(names, subprocess.run(["c++filt"] + names, capture_output=True, text=True).stdout.splitlines()))  # noqa: E731

counts, cur, arch = collections.OrderedDict(), None, set()
for line in sass.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        cur = m.group(1)
        counts[cur] = collections.Counter()
        continue
    m = re.search(r"arch = (sm_\w+)", line)
    if m:
        arch.add(m.group(1))
    m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
    if m and cur:
        op = m.group(1)
        counts[cur][op.split(".")[0]] += 1
        if op.startswith("IMAD.WIDE"):
            counts[cur]["IMAD.WIDE*"] += 1
regs = {}
for m in re.finditer(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+)", res):
    regs[m.group(1)] = (int(m.group(2)), int(m.group(3)), int(m.group(4)))
names = demangle(list(counts))
tot = collections.Counter()
for c in counts.values():
    tot.update(c)
print("# SASS excerpt of the shipped `libb200zk.so` (round 2)\n")
print(f"`cuobjdump -sass ethrex_b200/libb200zk.so`: arch {sorted(arch)}, {len(counts)} kernels / device functions; source hash `{bench.source_hash()}`"
      " (`bench.source_hash()`: csrc/*.cu, *.cuh, Makefile, include/b200zk.h).\n")
keys = ["IMAD.WIDE*", "IMAD", "IADD3", "UBLKCP", "SYNCS", "ATOMS", "ATOMG", "RED", "SHFL", "DFMA", "CALL", "LDG", "STG", "LDS", "STS", "BAR"]
print("Whole library: " + ", ".join(f"`{k}` x {tot[k]}" for k in keys) + ".")
tc = [k for k in tot if k.startswith(("UTC", "LDTM", "STTM", "HMMA", "HGMMA", "QGMMA", "IGMMA", "UTMALDG", "UTMASTG"))]
print(f"Tensor-core / TMEM / tensor-map mnemonics present: {tc or 'none'} -- as the north star prescribes for this path (256-bit modular integer arithmetic, no dense "
      "contraction); `UBLKCP` + `SYNCS` are the bulk-copy engine (cp.async.bulk + mbarrier) staging scalar tiles and NTT tiles.\n")
print("| kernel | registers | stack | static smem | `IMAD.WIDE*` | `IADD3` | `UBLKCP` | `SYNCS` | `SHFL` | `ATOMS` | `ATOMG`+`RED` | `CALL` | instructions |")
print("|---|---|---|---|---|---|---|---|---|---|---|---|---|")
want = ("msm_accumulate", "msm_sort", "msm_hist", "msm_scatter", "ntt_pass", "partial_tree", "bucket_chunk", "bucket_bit", "groth16_assemble", "fq_mul", "precompute_windows",
        "pairing_check", "bls_g1_decode", "msm_encode", "fr_quotient")
for f, c in counts.items():
    nm = names.get(f, f)
    if not any(w in nm for w in want):
        continue
    r = regs.get(f, ("", "", ""))
    short = re.sub(r"\(.*", "", nm).replace("b200zk::", "")
    short = short.replace("Fe<b200zk::FqCfg>", "Fq").replace("FeBig<b200zk::Fp381Cfg>", "Fp381").replace("Fe<FqCfg>", "Fq").replace("FeBig<Fp381Cfg>", "Fp381")
    print(f"| `{short}` | {r[0]} | {r[1]} | {r[2]} | {c['IMAD.WIDE*']} | {c['IADD3']} | {c['UBLKCP']} | {c['SYNCS']} | {c['SHFL']} | {c['ATOMS']} | {c['ATOMG'] + c['RED']} | {c['CALL']} | {sum(v for k, v in c.items() if k != 'IMAD.WIDE*')} |")
