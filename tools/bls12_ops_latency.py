"""Latency of the EIP-2537 addition and MSM calls on the device: b200zk_bls12_381_{g1,g2}_add_batch with 1 and 4096 items,
b200zk_bls12_381_{g1,g2}_msm_batch with one call of k = 1, 128 and 4096 pairs (G2: 2048), and 64 calls of k = 16.  Chain
bases P_i = (a + i d) G with random 256-bit scalars; every answer is checked against the closed form.  Wall-clock per call
(every call returns on the host with its results); medians over the steps after warm-up.  Prints one JSON line per case,
with the card's name and power limit read in the same run.

    python tools/bls12_ops_latency.py [--steps 5] [--warmup 1]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402

import bls12_ops_ref as ops  # noqa: E402
import ethrex_b200 as eb  # noqa: E402
from kzg_proof_latency import gpu_identity, wall_ms  # noqa: E402

A, D = 0x5EED, 0x1F1F1F


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
    rng = np.random.default_rng(2537)

    def emit(case, shape, t):
        print(json.dumps({"tool": "bls12_ops_latency", "gpu": ident, "case": case, "shape": shape, "steps": a.steps, "warmup": a.warmup,
                          "call_ms": t}), flush=True)
    for g, add, msm, large in ((ops.G1, ctx.bls12_381_g1_add_batch, ctx.bls12_381_g1_msm_batch, 4096),
                               (ops.G2, ctx.bls12_381_g2_add_batch, ctx.bls12_381_g2_msm_batch, 2048)):
        bases = g.chain(max(large, 4097), A, D)
        enc = [g.encode(p) for p in bases]
        sums = [g.encode(p) for p in g.chain(4096, 2 * A + D, 2 * D)]  # P_i + P_(i+1) = (2a + d + 2 i d) G
        for n in (1, 4096):
            want = b"".join(sums[:n])
            args = (b"".join(enc[:n]), b"".join(enc[1:n + 1]))
            emit(f"{g.name.lower()}_add_batch", {"items": n}, timed(lambda: add(*args), lambda o: o == (want, [0] * n), a.steps, a.warmup))
        for count, k in ((1, 1), (1, 128), (1, large), (64, 16)):
            ks = [[int.from_bytes(rng.bytes(32), "big") for _ in range(k)] for _ in range(count)]
            calls = [g.calldata(list(zip(bases[:k], s))) for s in ks]
            want = [g.encode(g.chain_msm(s, A, D)) for s in ks]
            emit(f"{g.name.lower()}_msm_batch", {"calls": count, "k": k}, timed(lambda: msm(calls), lambda o: o == (want, [0] * count), a.steps, a.warmup))
    ctx.close()


if __name__ == "__main__":
    main()
