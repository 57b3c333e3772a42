"""Latency of the EIP-2537 map-to-curve calls on the device: b200zk_bls12_381_map_fp_to_g1_batch and
b200zk_bls12_381_map_fp2_to_g2_batch with 1, 64 and 4096 random field elements.  Every answer is checked against the
RFC 9380 oracle (tests/bls12_map_ref.py).  Wall-clock per call (every call returns on the host with its results);
min / median / max over the steps after warm-up.  Prints one JSON line per case, with the card's name and power limit
read in the same run.

    python tools/bls12_map_latency.py [--steps 5] [--warmup 1]
"""
import argparse
import json
import os
import random
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    sys.path.insert(0, p)

import bls12_map_ref as M  # noqa: E402
import ethrex_b200 as eb  # noqa: E402
from kzg_proof_latency import gpu_identity, wall_ms  # noqa: E402


def timed(fn, check, steps, warmup):
    t = []
    for step in range(warmup + steps):
        ms, out = wall_ms(fn)
        check(out)
        if step >= warmup:
            t.append(ms)
    return {"min": min(t), "median": statistics.median(t), "max": max(t)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    ctx = eb.Context(0)
    ident = gpu_identity(0)
    rng = random.Random(2537)
    cases = (("map_fp_to_g1_batch", ctx.bls12_381_map_fp_to_g1_batch, lambda: M.fp64(rng.randrange(M.P)), M.map_fp_to_g1_bytes),
             ("map_fp2_to_g2_batch", ctx.bls12_381_map_fp2_to_g2_batch, lambda: M.fp2_64((rng.randrange(M.P), rng.randrange(M.P))),
              M.map_fp2_to_g2_bytes))
    for name, fn, draw, oracle in cases:
        encs = [draw() for _ in range(4096)]
        want = [oracle(e) for e in encs]
        for n in (1, 64, 4096):
            data = b"".join(encs[:n])
            exp = (b"".join(o for o, _ in want[:n]), [s for _, s in want[:n]])
            t = timed(lambda: fn(data), lambda o: o == exp, a.steps, a.warmup)
            print(json.dumps({"tool": "bls12_map_latency", "gpu": ident, "case": name, "shape": {"items": n}, "steps": a.steps,
                              "warmup": a.warmup, "call_ms": t}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
