"""Latency of KZG verification and the BLS12-381 pairing check on the device: b200zk_kzg_verify_proof_batch at n items,
b200zk_kzg_verify_blob_proof_batch at n blobs, b200zk_bls12_381_pairing_check_batch with n two-pair checks.  Synthetic
known-tau setup; every input is valid and every answer is checked.  Wall-clock per call (every call returns on the host
with its results); medians over the steps after warm-up.  Prints one JSON line per case, with the card's name and power
limit read in the same run.

    python tools/kzg_verify_latency.py [--steps 5] [--warmup 1]
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

import bls_pairing_ref as B  # noqa: E402
import bls_ref as bls  # noqa: E402
import ethrex_b200 as eb  # noqa: E402
import kzg_ref as ref  # noqa: E402
from kzg_proof_latency import gpu_identity, wall_ms  # noqa: E402

TAU = 0x2F1B7C93D4A5E6F708192A3B4C5D6E7F8091A2B3C4D5E6F708192A3B4C5D6E7F % bls.R


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
    g1 = ctx.bls12_381_g1_bases_upload(b"".join(bls.compress(p) for p in bls.generator_multiples(bls.lagrange_setup_scalars(TAU))), 4096)
    ctx.bases_precompute(g1, 0)
    g2 = ctx.bls12_381_g2_bases_upload(B.G2_COMPRESSED + B.g2_compress(B.g2_mul(TAU, B.G2)), 2)
    rng = np.random.default_rng(4844)
    blobs = [ref.to_blob([int.from_bytes(rng.bytes(32), "big") % bls.R for _ in range(4096)]) for _ in range(9)]
    cs, ps = ctx.kzg_blob_to_commitment_and_proof(g1, b"".join(blobs))
    ys = [ref.quotient(ref.blob_values(b), ref.challenge(b, c))[1] for b, c in zip(blobs, cs)]
    items = [(c, ref.challenge(b, c).to_bytes(32, "big"), y.to_bytes(32, "big"), p) for b, c, p, y in zip(blobs, cs, ps, ys)]

    def emit(case, n, t):
        print(json.dumps({"tool": "kzg_verify_latency", "gpu": ident, "case": case, "n": n, "steps": a.steps, "warmup": a.warmup, "call_ms": t}), flush=True)
    for n in (1, 64, 4096):
        batch = [items[i % len(items)] for i in range(n)]
        args = [b"".join(it[k] for it in batch) for k in range(4)]
        emit("kzg_verify_proof_batch", n, timed(lambda: ctx.kzg_verify_proof_batch(g2, *args), lambda o: o == ([1] * n, [0] * n), a.steps, a.warmup))
    for n in (1, 6, 9):
        args = (b"".join(blobs[:n]), b"".join(cs[:n]), b"".join(ps[:n]))
        emit("kzg_verify_blob_proof_batch", n, timed(lambda: ctx.kzg_verify_blob_proof_batch(g2, *args), lambda o: o is True, a.steps, a.warmup))
    check = B.g1_eip2537(B.G1) + B.g2_eip2537(B.G2) + B.g1_eip2537(B.G1) + B.g2_eip2537(B.g2_neg(B.G2))
    for n in (1, 1024):
        emit("bls12_381_pairing_check_batch", n, timed(lambda: ctx.bls12_381_pairing_check_batch([check] * n), lambda o: o == ([1] * n, [0] * n), a.steps, a.warmup))
    ctx.bases_free(g1)
    ctx.bases_free(g2)
    ctx.close()


if __name__ == "__main__":
    main()
