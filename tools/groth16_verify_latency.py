"""Latency of Groth16 batch verification on the device (b200zk_groth16_verify_batch) beside the per-proof route it
replaces (each proof's ecpairing calldata, with one b200zk_g1_msm call for its public inputs, then one
b200zk_bn254_pairing_check_batch over the N four-pair checks), both in the same run, for N in {1, 16, 256, 4096} and
n_pub in {2, 8}; and the batch call on a batch with one bad proof (C swapped in from another proof), which takes the
failure path.  Proofs are simulated from known toxic waste (tests/groth16_batch_ref.py), each with its own A, B and C.
Every verdict is checked.  Wall-clock per call (every call returns on the host with its verdicts); min / median / max over
the steps after warm-up.  Prints one JSON line per case, with the card's name and power limit read in the same run.

    python tools/groth16_verify_latency.py [--steps 5] [--warmup 1] [--sizes 1,16,256,4096]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    sys.path.insert(0, p)
import ethrex_b200 as eb  # noqa: E402
import groth16_batch_ref as ref  # noqa: E402
from ethrex_b200.groth16 import Groth16Verifier  # noqa: E402
from kzg_proof_latency import gpu_identity  # noqa: E402
from kzg_verify_latency import timed  # noqa: E402


def per_proof_route(ctx, ver, proofs, xs):
    """the route Groth16Verifier.verify_batch took before the batch call: calldata() per proof, one pairing-check batch"""
    cds = [ver.calldata(p, x) for p, x in zip(proofs, xs)]
    res, st = ctx.bn254_pairing_check_batch(cds)
    return [bool(r) and s == 0 for r, s in zip(res, st)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--sizes", default="1,16,256,4096")
    a = ap.parse_args()
    sizes = [int(s) for s in a.sizes.split(",")]
    ctx = eb.Context(0)
    ident = gpu_identity(0)

    def emit(case, extra, t):
        print(json.dumps({"tool": "groth16_verify_latency", "gpu": ident, "case": case, **extra, "steps": a.steps, "warmup": a.warmup,
                          "call_ms": t}), flush=True)

    for n_pub in (2, 8):
        key = ref.SimKey(n_pub, seed=0x6716 + n_pub)
        items = [key.proof() for _ in range(max(sizes))]
        ver = Groth16Verifier(ctx, *key.elements())
        for n in sizes:
            proofs, xs = [p for p, _ in items[:n]], [x for _, x in items[:n]]
            xb = b"".join(int(v).to_bytes(32, "big") for x in xs for v in x)
            extra = {"n": n, "n_pub": n_pub}

            def all_valid(out):
                if out != ([True] * n, [0] * n, True):
                    raise SystemExit(f"a valid batch of {n} was not decided valid by the combined check")

            def all_true(out):
                if out != [True] * n:
                    raise SystemExit(f"the per-proof route refused a valid batch of {n}")

            emit("groth16_verify_batch", extra, timed(lambda: ctx.groth16_verify_batch(key.vk, proofs, xb), all_valid, a.steps, a.warmup))
            emit("per_proof_route", extra, timed(lambda: per_proof_route(ctx, ver, proofs, xs), all_true, a.steps, a.warmup))
            if n > 1:
                k = n // 2
                bad = list(proofs)
                bad[k] = bad[k][:192] + proofs[k - 1][192:]
                want = [i != k for i in range(n)]

                def one_bad(out):
                    if out[0] != want or out[2]:
                        raise SystemExit(f"the failure path gave wrong verdicts for a batch of {n}")

                emit("groth16_verify_batch_one_bad", extra, timed(lambda: ctx.groth16_verify_batch(key.vk, bad, xb), one_bad, a.steps, a.warmup))
    ctx.close()


if __name__ == "__main__":
    main()
