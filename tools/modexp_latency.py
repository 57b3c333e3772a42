"""Latency and throughput of b200zk_modexp_batch (MODEXP, precompile 0x05) on the device, for the three shapes callers
use: 32/32/32-byte items (field inversions and square roots in on-chain SNARK verifiers) x1, x4096 and x65536; RSA-2048
and RSA-4096 signature checks with e = 65537 x1 and x1024; and the EIP-7823 worst case, 1024/1024/1024-byte items,
x1, x132 (one per SM) and x1056.  Wall-clock per call (the call returns on the host with its results: upload, kernels,
download); medians over the steps after warm-up.  Every answer is checked against Python's `pow`.

The only CPU comparator on the host is CPython's own `pow` (not malachite, which the reference uses), one thread, over
the same items: all of them for the small shapes, and the first few of the worst case with the per-item time scaled to
the count ("cpu_items_timed" says how many).  Prints one JSON line per case, with the card's name and power limit read
in the same run.

    python tools/modexp_latency.py [--steps 5] [--warmup 1]
"""
import argparse
import json
import os
import random
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    sys.path.insert(0, p)

import ethrex_b200 as eb  # noqa: E402
import modexp_ref as ref  # noqa: E402
from kzg_proof_latency import gpu_identity, wall_ms  # noqa: E402


def cases(rng):
    """(name, unique items, counts, items CPython times at most)"""
    small = [ref.rand_item(rng, 32, exp_len=32) for _ in range(4096)]
    rsa2048, _ = ref.rsa_items(rng, 2048, 256)
    rsa4096, _ = ref.rsa_items(rng, 4096, 256)
    worst = [tuple(ref.rand_bytes(rng, 1024) for _ in range(3)) for _ in range(132)]
    return [("32/32/32", small, (1, 4096, 65536), 65536), ("rsa2048_e65537", rsa2048, (1, 1024), 1024),
            ("rsa4096_e65537", rsa4096, (1, 1024), 1024), ("1024/1024/1024", worst, (1, 132, 1056), 4)]


def cpython_ms(items, cap):
    """CPython pow over the first min(len, cap) items, scaled to all of them"""
    timed = items[:cap]
    t0 = time.perf_counter()
    for it in timed:
        ref.modexp(*it)
    per = (time.perf_counter() - t0) * 1e3 / len(timed)
    return per * len(items), len(timed)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    ctx = eb.Context(0)
    ident = gpu_identity(0)
    print(json.dumps({"tool": "modexp_latency", "gpu": ident, "cpu_baseline": "CPython pow, 1 thread"}), flush=True)
    for name, unique, counts, cap in cases(random.Random(5)):
        want = [ref.modexp(*it) for it in unique]
        for count in counts:
            items = [unique[i % len(unique)] for i in range(count)]
            t = []
            for step in range(a.warmup + a.steps):
                ms, (outs, st) = wall_ms(lambda: ctx.modexp_batch(items))
                assert st == [0] * count and all(o == want[i % len(unique)] for i, o in enumerate(outs)), f"{name} x{count}: wrong result"
                if step >= a.warmup:
                    t.append(ms)
            med = statistics.median(t)
            cpu, timed = cpython_ms(items, cap)
            print(json.dumps({"tool": "modexp_latency", "gpu": ident, "case": name, "count": count, "steps": a.steps, "warmup": a.warmup,
                              "call_ms": {"min": min(t), "median": med, "max": max(t)}, "items_per_s": count / (med / 1e3),
                              "cpython_ms": cpu, "cpu_items_timed": timed}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
