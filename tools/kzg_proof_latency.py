"""Latency of EIP-4844 blob proofs: one b200zk_kzg_blob_to_commitment_and_proof call for a batch of 1, 6 and 9 blobs over
a synthetic 4096-point setup (plain bases, then a window table), against the path it replaces in the same process -- per
blob, the commitment MSM, the challenge hashed in Python, the quotient in Python big integers (tests/kzg_ref.py) and a
second MSM call.  Wall-clock per call (every call returns on the host with its results).  Prints one JSON line per
(setup, batch size), with the card's name and power limit.

    python tools/kzg_proof_latency.py [--blobs 1 6 9] [--steps 5] [--warmup 1]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import bls_ref as bls  # noqa: E402
import ethrex_b200 as eb  # noqa: E402
import kzg_ref as ref  # noqa: E402


def gpu_identity(index: int = 0) -> dict:
    try:
        out = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30, check=True).stdout.strip()
        name, watts = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit_w": float(watts)}
    except Exception:
        return {"name": torch.cuda.get_device_name(index), "power_limit_w": None}


def wall_ms(fn):
    t0 = time.perf_counter()
    out = fn()
    return (time.perf_counter() - t0) * 1e3, out


def old_path(ctx, h, blobs):
    """per blob: commitment MSM, hashlib challenge, host big-integer quotient, proof MSM"""
    out = []
    for blob in blobs:
        c = ctx.kzg_blob_to_commitment(h, blob)[0]
        q, _ = ref.quotient(ref.blob_values(blob), ref.challenge(blob, c))
        out.append((c, ctx.bls12_381_g1_msm_resident(h, ref.to_blob(q), 4096)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blobs", type=int, nargs="+", default=[1, 6, 9])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    ctx = eb.Context(0)
    ident = gpu_identity(0)
    rng = np.random.default_rng(4844)
    pool = [ref.to_blob([int.from_bytes(rng.bytes(32), "big") % bls.R for _ in range(4096)]) for _ in range(max(a.blobs))]
    setup = bls.chain(4096, 0x1234567, 0x9E3779B97F4A7C15)  # P_i = (k + i d) G, uncompressed
    for table in (False, True):
        h = ctx.bls12_381_g1_bases_upload(setup, 4096, 0)
        if table:
            ctx.bases_precompute(h, 0)
        for n in a.blobs:
            blobs = pool[:n]
            batch = b"".join(blobs)
            new, old = [], []
            for step in range(a.warmup + a.steps):
                t_new, (cs, ps) = wall_ms(lambda: ctx.kzg_blob_to_commitment_and_proof(h, batch))
                t_old, pairs = wall_ms(lambda: old_path(ctx, h, blobs))
                assert pairs == list(zip(cs, ps)), "the two paths disagree"
                if step >= a.warmup:
                    new.append(t_new)
                    old.append(t_old)
            print(json.dumps({"tool": "kzg_proof_latency", "gpu": ident, "setup": "window_table" if table else "plain", "blobs": n,
                              "steps": a.steps, "warmup": a.warmup,
                              "device_call_ms": {"min": min(new), "median": statistics.median(new), "max": max(new)},
                              "host_quotient_path_ms": {"min": min(old), "median": statistics.median(old), "max": max(old)}}), flush=True)
        ctx.bases_free(h)
    ctx.close()


if __name__ == "__main__":
    main()
