"""Latency of EIP-7594 cell recovery on the device: b200zk_kzg_recover_cells_and_cell_proofs (all 128 cells and 128 cell
proofs per blob from a subset of its cells) for 1, 6, 21 and 72 blobs, given exactly 64 cells and given 96 cells per blob.
Synthetic known-tau setup; every call's output is compared with what b200zk_kzg_compute_cells and
b200zk_kzg_blob_to_commitment_and_cell_proofs return for the same blobs.  Wall-clock per call (every call returns on the
host with its results): median, min and max over the steps after warm-up.  A per-phase split comes from one profiled call
per case (torch.profiler's CUDA kernel times, summed per phase): the recovery kernels (kzg_recover_blob: coefficients and
blob from 64 cells; kzg_recover_check: every given cell against the rebuilt ones), the extension (kzg_cells_extend), the
input range check, and the FK20 phases the call shares with the cell-proof call.  Prints one JSON line per case with the
card's name and power limit read in the same run.

    python tools/kzg_recover_latency.py [--steps 5] [--warmup 1]
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
import torch  # noqa: E402

import bls_ref as bls  # noqa: E402
import ethrex_b200 as eb  # noqa: E402
import kzg_cells_ref as ref  # noqa: E402
import kzg_ref  # noqa: E402
from kzg_proof_latency import gpu_identity  # noqa: E402
from kzg_verify_latency import timed  # noqa: E402

TAU = 0x2F1B7C93D4A5E6F708192A3B4C5D6E7F8091A2B3C4D5E6F708192A3B4C5D6E7F % bls.R
DISTINCT = 6  # batches repeat 6 random blobs
PHASES = {"kzg_recover_blob": "recover_coefficients_and_blob", "kzg_recover_check": "consistency_check", "kzg_cells_extend": "extension",
          "kzg_fk20_columns": "fk20_coefficients_and_fr_dfts", "kzg_fk20_msm": "fk20_msms", "kzg_fk20_proofs": "fk20_g1_dfts",
          "bls_scalar_check": "input_check"}


def phase_split(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA or "memcpy" in ev.name.lower() or "memset" in ev.name.lower():
            continue
        phase = next((v for k, v in PHASES.items() if k in ev.name), "other")
        out[phase] = out.get(phase, 0.0) + ev.device_time / 1000.0
    return {k: round(v, 3) for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    ctx = eb.Context(0)
    ident = gpu_identity(0)
    lag = ctx.bls12_381_g1_bases_upload(b"".join(bls.compress(p) for p in bls.generator_multiples(bls.lagrange_setup_scalars(TAU))), 4096)
    mono = ctx.bls12_381_g1_bases_upload(b"".join(bls.compress(p) for p in bls.generator_multiples([pow(TAU, i, bls.R) for i in range(4096)])), 4096)
    rng = np.random.default_rng(7594)
    blobs = [kzg_ref.to_blob([int.from_bytes(rng.bytes(32), "big") % bls.R for _ in range(4096)]) for _ in range(DISTINCT)]
    cells = ctx.kzg_compute_cells(b"".join(blobs))
    assert cells[0] == ref.compute_cells(blobs[0])
    proofs = ctx.kzg_blob_to_commitment_and_cell_proofs(lag, mono, b"".join(blobs))[1]
    pick = random.Random(7594)

    for given in (64, 96):
        for n in (1, 6, 21, 72):
            idx = [i % DISTINCT for i in range(n)]
            items = []
            for i in idx:
                ix = pick.sample(range(128), given)
                items.append((ix, [cells[i][c] for c in ix]))
            want = ([c for i in idx for c in cells[i]], [p for i in idx for p in proofs[128 * i:128 * i + 128]])

            def check(o):
                assert o == want

            def call():
                return ctx.kzg_recover_cells_and_cell_proofs(mono, items)

            t = timed(call, check, a.steps, a.warmup)
            print(json.dumps({"tool": "kzg_recover_latency", "gpu": ident, "case": "kzg_recover_cells_and_cell_proofs", "n_blobs": n,
                              "cells_given": given, "steps": a.steps, "warmup": a.warmup, "call_ms": t,
                              "kernel_ms": phase_split(lambda: check(call()))}), flush=True)
    for h in (lag, mono):
        ctx.bases_free(h)
    ctx.close()


if __name__ == "__main__":
    main()
