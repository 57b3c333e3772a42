"""ncu `--page raw --csv` capture of tools/profile_workload.py -> profiles/r2_ncu_kernels.json, the file bench.py reads its
`roofline.traffic` / `fmaheavy` side fields from.  The JSON records the hash of the sources it was captured on
(bench.source_hash); bench.py ignores it when the tree has changed since.

    python tools/ncu_to_profile_json.py gpurun_out/r2_ncu_full.csv [profiles/r2_ncu_kernels.json]
"""
import csv
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WANT = {
    "dram__bytes_read.sum": "dram_bytes_read",
    "dram__bytes_write.sum": "dram_bytes_write",
    "gpu__time_duration.sum": "duration",
    "sm__pipe_fmaheavy_cycles_active.avg.pct_of_peak_sustained_active": "fmaheavy_pct",
    "sm__pipe_fmaheavy_cycles_active.avg.pct_of_peak_sustained_elapsed": "fmaheavy_pct_elapsed",
    "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active": "alu_pct",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed": "sm_throughput_pct",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed": "dram_throughput_pct",
    "lts__t_sector_hit_rate.pct": "l2_hit_pct",
    "sm__warps_active.avg.pct_of_peak_sustained_active": "warps_active_pct",
    "launch__registers_per_thread": "registers",
    "launch__grid_size": "grid",
    "launch__block_size": "block",
    "smsp__inst_executed.sum": "instructions",
}
UNIT_SCALE = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "ns": 1e-6, "us": 1e-3, "ms": 1.0, "s": 1e3, "nsecond": 1e-6, "usecond": 1e-3, "msecond": 1.0, "second": 1e3}


def read_rows(path):
    with open(path, newline="") as f:
        lines = [ln for ln in f if not ln.startswith("==")]
    rd = list(csv.reader(lines))
    hdr_i = next(i for i, r in enumerate(rd) if "Kernel Name" in r)
    hdr, units = rd[hdr_i], rd[hdr_i + 1]
    out = []
    for r in rd[hdr_i + 2:]:
        if len(r) != len(hdr):
            continue
        row = {"kernel": r[hdr.index("Kernel Name")]}
        for col, key in WANT.items():
            if col in hdr:
                j = hdr.index(col)
                try:
                    v = float(r[j].replace(",", ""))
                except ValueError:
                    continue
                if v != v:  # nan ("n/a" for a metric the kernel does not exercise)
                    continue
                row[key] = v * UNIT_SCALE.get(units[j], 1.0)
        out.append(row)
    return out


def main():
    import bench
    src = sys.argv[1]
    dst = sys.argv[2] if len(sys.argv) > 2 else os.path.join(ROOT, "profiles", "r2_ncu_kernels.json")
    rows = read_rows(src)
    kernels = {}

    def last(pred):
        m = [r for r in rows if pred(r["kernel"])]
        return m[-1] if m else None

    g1 = last(lambda k: "msm_accumulate<" in k and "Fq2" not in k and "Fp381" not in k)
    g2 = last(lambda k: "msm_accumulate_g2_pair" in k or ("msm_accumulate<" in k and "Fq2" in k))
    if g1:
        kernels["msm_accumulate_g1"] = g1
    if g2:
        kernels["msm_accumulate_g2"] = g2
    for name in ("msm_hist", "msm_scatter", "msm_sort_count", "msm_sort_coarse", "msm_sort_fine"):
        r = last(lambda k, name=name: k.startswith(name) or (" " + name) in k or ("::" + name) in k)
        if r:
            kernels[name] = r
    ntt = [r for r in rows if "ntt_pass" in r["kernel"]]
    if ntt:
        passes = ntt[-(len(ntt) // 2):] if len(ntt) % 2 == 0 else ntt  # the workload runs the transform twice: keep the second
        tot = {"kernel": "ntt_pass x %d (one forward 2^24 transform)" % len(passes), "passes": passes}
        for key in ("dram_bytes_read", "dram_bytes_write", "duration", "instructions"):
            if all(key in p for p in passes):
                tot[key] = sum(p[key] for p in passes)
        for key in ("fmaheavy_pct", "fmaheavy_pct_elapsed"):
            if all(key in p and "duration" in p for p in passes):
                tot[key] = sum(p[key] * p["duration"] for p in passes) / sum(p["duration"] for p in passes)
        kernels["ntt_forward_2_24"] = tot
    doc = {"source_hash": bench.source_hash(), "captured_from": os.path.basename(src),
           "how": "ncu --set full --clock-control none python tools/profile_workload.py (2^24 G1 MSM, G2 MSM over window tables, forward NTT); durations in ms, "
                  "cold-cache and serialised: use shares and percentages, not absolutes",
           "kernels": kernels}
    os.makedirs(os.path.dirname(os.path.abspath(dst)), exist_ok=True)
    with open(dst, "w") as f:
        json.dump(doc, f, indent=1)
    for k, v in kernels.items():
        print(k, {x: v[x] for x in ("duration", "dram_bytes_read", "dram_bytes_write", "fmaheavy_pct", "fmaheavy_pct_elapsed", "registers") if x in v})


if __name__ == "__main__":
    main()
