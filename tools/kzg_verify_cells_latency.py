"""Latency of EIP-7594 cell-proof verification over arbitrary cells on the device (b200zk_kzg_verify_cells): one data
column of 6, 21 and 72 blobs, a slot's samples (8 columns of 21 blobs) and every cell of 21 blobs, the last beside
b200zk_kzg_verify_cell_proof_batch on the same blobs.  Synthetic known-tau setup; the blobs are distinct, and their
cells and proofs come from the device's compute_cells and FK20 calls, so the number of distinct commitments is the
number of blobs.  Every answer is checked.  Wall-clock per call (every call returns on the host with its answer);
medians over the steps after warm-up.  Prints one JSON line per case, with the card's name and power limit read in the
same run.  No CPU baseline: c-kzg is not installed where this runs.

    python tools/kzg_verify_cells_latency.py [--steps 5] [--warmup 1]
"""
import argparse
import json
import os
import random
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
N_BLOBS = 72


def must_verify(out):
    if out is not True:
        raise SystemExit("an honest set of cells did not verify")


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
    mono = ctx.bls12_381_g1_bases_upload(b"".join(bls.compress(p) for p in bls.generator_multiples([pow(TAU, i, bls.R) for i in range(4096)])), 4096)
    rng = np.random.default_rng(7594)
    blobs = [kzg_ref.to_blob([int.from_bytes(rng.bytes(32), "big") % bls.R for _ in range(4096)]) for _ in range(N_BLOBS)]
    cells = ctx.kzg_compute_cells(b"".join(blobs))
    cs, ps = ctx.kzg_blob_to_commitment_and_cell_proofs(g1, mono, b"".join(blobs))
    assert len(set(cs)) == N_BLOBS

    def emit(case, extra, t):
        print(json.dumps({"tool": "kzg_verify_cells_latency", "gpu": ident, "case": case, **extra, "steps": a.steps, "warmup": a.warmup,
                          "call_ms": t, "cpu_baseline": "not measured (no c-kzg)"}), flush=True)

    pick = random.Random(7594)
    cases = [(1, 6), (1, 21), (1, 72), (8, 21), (128, 21)]
    for n_cols, n_blobs in cases:
        cols = sorted(pick.sample(range(128), n_cols))
        pairs = [(b, c) for b in range(n_blobs) for c in cols]
        args = (b"".join(cs[b] for b, _ in pairs), [c for _, c in pairs], b"".join(cells[b][c] for b, c in pairs),
                b"".join(ps[128 * b + c] for b, c in pairs))
        extra = {"columns": n_cols, "n_blobs": n_blobs, "n_cells": len(pairs), "n_commitments": len({b for b, _ in pairs})}
        emit("kzg_verify_cells", extra, timed(lambda: ctx.kzg_verify_cells(g1, g2, *args), must_verify, a.steps, a.warmup))
        if n_cols == 128:
            whole = (b"".join(blobs[:n_blobs]), b"".join(cs[:n_blobs]), b"".join(ps[:128 * n_blobs]))
            emit("kzg_verify_cell_proof_batch", extra,
                 timed(lambda: ctx.kzg_verify_cell_proof_batch(g1, g2, *whole), must_verify, a.steps, a.warmup))
    for h in (g1, g2, mono):
        ctx.bases_free(h)
    ctx.close()


if __name__ == "__main__":
    main()
