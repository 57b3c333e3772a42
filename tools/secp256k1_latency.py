"""Latency and throughput of b200zk_secp256k1_ecrecover_batch on the device: one call of count = 1, 256 (about one
block's transactions), 4096, 65536 and 2^20 signatures.  The items are 4096 distinct `cryptography` signatures over random
digests, repeated to fill the larger batches (every item is a full recovery; the device keeps nothing between items), and
every answer is checked against the signer's own key.  Wall-clock per call (the call returns on the host with its results:
upload, kernel, download); medians over the steps after warm-up, and recoveries per second at the median.  Prints one JSON
line per case, with the card's name and power limit read in the same run.

    python tools/secp256k1_latency.py [--steps 5] [--warmup 1]
"""
import argparse
import json
import os
import random
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    sys.path.insert(0, p)
from cryptography.hazmat.primitives import hashes  # noqa: E402
from cryptography.hazmat.primitives.asymmetric import ec, utils  # noqa: E402

import ethrex_b200 as eb  # noqa: E402
import secp256k1_ref as ref  # noqa: E402
from kzg_proof_latency import gpu_identity, wall_ms  # noqa: E402

UNIQUE = 4096


def signatures(rng, n):
    """n (sig, digest, keccak256 of the signer's key); recid from the public key's point (the oracle picks it)"""
    out = []
    for _ in range(n):
        key = ec.derive_private_key(rng.randrange(1, ref.N), ec.SECP256K1())
        digest = rng.randbytes(32)
        r, s = utils.decode_dss_signature(key.sign(digest, ec.ECDSA(utils.Prehashed(hashes.SHA256()))))
        pub = key.public_key().public_numbers()
        want = ref.address_hash((pub.x, pub.y))
        sig = r.to_bytes(32, "big") + s.to_bytes(32, "big") + b"\0"
        if ref.recover(sig, digest) != (ref.OK, want):
            sig = sig[:64] + b"\1"
        out.append((sig, digest, want))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--counts", default="1,256,4096,65536,1048576")
    a = ap.parse_args()
    items = signatures(random.Random(256), UNIQUE)
    sigs = b"".join(s for s, _, _ in items)
    msgs = b"".join(m for _, m, _ in items)
    want = b"".join(w for _, _, w in items)
    ctx = eb.Context(0)
    ident = gpu_identity(0)
    for count in (int(c) for c in a.counts.split(",")):
        reps, rem = divmod(count, UNIQUE)
        s_in = sigs * reps + sigs[:65 * rem]
        m_in = msgs * reps + msgs[:32 * rem]
        expect = (want * reps + want[:32 * rem], [0] * count)
        t = []
        for step in range(a.warmup + a.steps):
            ms, res = wall_ms(lambda: ctx.secp256k1_ecrecover_batch(s_in, m_in, low_s=False))
            assert res == expect, f"count {count}: device output differs from the signers' keys"
            if step >= a.warmup:
                t.append(ms)
        med = statistics.median(t)
        print(json.dumps({"tool": "secp256k1_latency", "gpu": ident, "count": count, "steps": a.steps, "warmup": a.warmup,
                          "call_ms": {"min": min(t), "median": med, "max": max(t)}, "recoveries_per_s": count / (med / 1e3)}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
