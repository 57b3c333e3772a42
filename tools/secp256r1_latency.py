"""Latency and throughput of b200zk_secp256r1_verify_batch (P256VERIFY, EIP-7951) on the device: one call of count = 1,
256, 4096, 65536 and 2^20 items.  The items are 4096 distinct OpenSSL signatures (through the `cryptography` package)
over random digests, repeated to fill the larger batches (every item is a full verification; the device keeps nothing
between items), and every answer is checked (all verify).  Wall-clock per call (the call returns on the host with its
results: upload, kernel, download); medians over the steps after warm-up, and verifications per second at the median.
The same run measures the single-thread rate of `cryptography`'s own P-256 verify on the host CPU as a baseline.  Prints
one JSON line per case, with the card's name and power limit read in the same run.

    python tools/secp256r1_latency.py [--steps 5] [--warmup 1]
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
from cryptography.hazmat.primitives import hashes  # noqa: E402
from cryptography.hazmat.primitives.asymmetric import ec, utils  # noqa: E402

import ethrex_b200 as eb  # noqa: E402
import secp256r1_ref as ref  # noqa: E402
from kzg_proof_latency import gpu_identity, wall_ms  # noqa: E402

UNIQUE = 4096


def signatures(rng, n):
    """n (160-byte input, public key object, DER signature, digest)"""
    out = []
    for _ in range(n):
        key = ec.derive_private_key(rng.randrange(1, ref.N), ec.SECP256R1())
        digest = rng.randbytes(32)
        der = key.sign(digest, ec.ECDSA(utils.Prehashed(hashes.SHA256())))
        r, s = utils.decode_dss_signature(der)
        pub = key.public_key()
        nums = pub.public_numbers()
        out.append((ref.encode(int.from_bytes(digest, "big"), r, s, (nums.x, nums.y)), pub, der, digest))
    return out


def cpu_rate(items, seconds=2.0):
    """single-thread verifications per second of `cryptography` (OpenSSL) over the same items, in the same process"""
    algo = ec.ECDSA(utils.Prehashed(hashes.SHA256()))
    done, t0 = 0, time.perf_counter()
    while time.perf_counter() - t0 < seconds:
        for _, pub, der, digest in items[:256]:
            pub.verify(der, digest, algo)
        done += 256
    return done / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--counts", default="1,256,4096,65536,1048576")
    a = ap.parse_args()
    items = signatures(random.Random(256), UNIQUE)
    inputs = b"".join(x for x, _, _, _ in items)
    ctx = eb.Context(0)
    ident = gpu_identity(0)
    print(json.dumps({"tool": "secp256r1_latency", "gpu": ident, "cpu_baseline": "cryptography (OpenSSL) P-256 verify, 1 thread",
                      "cpu_verifications_per_s": cpu_rate(items)}), flush=True)
    for count in (int(c) for c in a.counts.split(",")):
        reps, rem = divmod(count, UNIQUE)
        blob = inputs * reps + inputs[:160 * rem]
        t = []
        for step in range(a.warmup + a.steps):
            ms, res = wall_ms(lambda: ctx.secp256r1_verify_batch(blob))
            assert res == [True] * count, f"count {count}: a valid signature did not verify"
            if step >= a.warmup:
                t.append(ms)
        med = statistics.median(t)
        print(json.dumps({"tool": "secp256r1_latency", "gpu": ident, "count": count, "steps": a.steps, "warmup": a.warmup,
                          "call_ms": {"min": min(t), "median": med, "max": max(t)}, "verifications_per_s": count / (med / 1e3)}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
