"""Latency of EIP-7594 cell verification on the device: b200zk_kzg_verify_cell_proof_batch over whole blob bundles of 1, 6,
21 and 72 blobs (one transaction's cap, a full Osaka-era block, a sync batch), and b200zk_kzg_compute_cells at the same
sizes.  Synthetic known-tau setup, proofs from tests/kzg_cells_ref.py; every input is valid and every answer is checked.
Wall-clock per call (every call returns on the host with its results); medians over the steps after warm-up.  Prints one
JSON line per case, with the card's name and power limit read in the same run.  No CPU baseline: c-kzg is not installed
where this runs, so the CPU's time for the same call is not measured.

    python tools/kzg_cell_verify_latency.py [--steps 5] [--warmup 1]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402

import bls_ref as bls  # noqa: E402
import ethrex_b200 as eb  # noqa: E402
import kzg_cells_ref as ref  # noqa: E402
import kzg_ref  # noqa: E402
from kzg_proof_latency import gpu_identity  # noqa: E402
from kzg_verify_latency import timed  # noqa: E402

TAU = 0x2F1B7C93D4A5E6F708192A3B4C5D6E7F8091A2B3C4D5E6F708192A3B4C5D6E7F % bls.R
DISTINCT = 6  # bundles repeat 6 proven blobs: proving in Python costs about a second per blob


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    ctx = eb.Context(0)
    ident = gpu_identity(0)
    g1 = ctx.bls12_381_g1_bases_upload(b"".join(bls.compress(p) for p in bls.generator_multiples(bls.lagrange_setup_scalars(TAU))), 4096)
    ctx.bases_precompute(g1, 0)
    g2 = ctx.bls12_381_g2_bases_upload(ref.g2_setup(TAU), 65)
    rng = np.random.default_rng(7594)
    blobs = [kzg_ref.to_blob([int.from_bytes(rng.bytes(32), "big") % bls.R for _ in range(4096)]) for _ in range(DISTINCT)]
    cs, ps = ref.bundle(blobs, TAU)
    cells0 = ref.compute_cells(blobs[0])

    def emit(case, n, t):
        print(json.dumps({"tool": "kzg_cell_verify_latency", "gpu": ident, "case": case, "n_blobs": n, "steps": a.steps, "warmup": a.warmup,
                          "call_ms": t, "cpu_baseline": "not measured (no c-kzg)"}), flush=True)
    for n in (1, 6, 21, 72):
        idx = [i % DISTINCT for i in range(n)]
        args = (b"".join(blobs[i] for i in idx), b"".join(cs[i] for i in idx), b"".join(b"".join(ps[128 * i:128 * i + 128]) for i in idx))
        emit("kzg_verify_cell_proof_batch", n, timed(lambda: ctx.kzg_verify_cell_proof_batch(g1, g2, *args), lambda o: o is True, a.steps, a.warmup))
        emit("kzg_compute_cells", n, timed(lambda: ctx.kzg_compute_cells(args[0]), lambda o: len(o) == n and o[0] == cells0, a.steps, a.warmup))
    ctx.bases_free(g1)
    ctx.bases_free(g2)
    ctx.close()


if __name__ == "__main__":
    main()
