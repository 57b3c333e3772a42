"""Latency of EIP-7594 cell proofs on the device: b200zk_kzg_blob_to_commitment_and_cell_proofs (the commitment and 128 cell
proofs per blob, FK20) for 1, 6, 21 and 72 blobs.  Synthetic known-tau setup; every call's output is compared with
tests/kzg_cells_ref.py's bundle.  Wall-clock per call (every call returns on the host with its results): median, min and max
over the steps after warm-up.  The first call on a fresh monomial handle, which also builds its FK20 table, is reported
separately.  A per-phase split comes from one profiled call per size (torch.profiler's CUDA kernel times, summed per phase):
coefficients + column DFTs (one kernel, kzg_fk20_columns), the 64-term MSMs, the two G1 DFTs with the compression, and the
commitment MSMs (every other kernel of the call).  Prints one JSON line per case with the card's name and power limit read
in the same run.  No CPU baseline: c-kzg is not installed where this runs, so the CPU's time for the same call is not
measured.

    python tools/kzg_cell_proof_latency.py [--steps 5] [--warmup 1]
"""
import argparse
import json
import os
import sys
import time

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
DISTINCT = 6  # batches repeat 6 blobs whose bundles the Python oracle computed
PHASES = {"kzg_fk20_columns": "coefficients_and_fr_dfts", "kzg_fk20_msm": "msms", "kzg_fk20_proofs": "g1_dfts", "bls_scalar_check": "input_check"}


def phase_split(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA or "memcpy" in ev.name.lower() or "memset" in ev.name.lower():
            continue
        phase = next((v for k, v in PHASES.items() if k in ev.name), "commitment")
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
    ctx.bases_precompute(lag, 0)
    monomial = b"".join(bls.compress(p) for p in bls.generator_multiples([pow(TAU, i, bls.R) for i in range(4096)]))
    mono = ctx.bls12_381_g1_bases_upload(monomial, 4096)
    rng = np.random.default_rng(7594)
    blobs = [kzg_ref.to_blob([int.from_bytes(rng.bytes(32), "big") % bls.R for _ in range(4096)]) for _ in range(DISTINCT)]
    cs, ps = ref.bundle(blobs, TAU)

    def emit(case, n, **kw):
        print(json.dumps({"tool": "kzg_cell_proof_latency", "gpu": ident, "case": case, "n_blobs": n, "steps": a.steps, "warmup": a.warmup,
                          **kw, "cpu_baseline": "not measured (no c-kzg)"}), flush=True)

    t0 = time.perf_counter()
    out = ctx.kzg_blob_to_commitment_and_cell_proofs(lag, mono, blobs[0])
    first = (time.perf_counter() - t0) * 1e3
    assert out == ([cs[0]], ps[:128])
    emit("first_call_with_table_build", 1, call_ms=round(first, 3))
    for n in (1, 6, 21, 72):
        idx = [i % DISTINCT for i in range(n)]
        want = ([cs[i] for i in idx], [p for i in idx for p in ps[128 * i:128 * i + 128]])
        data = b"".join(blobs[i] for i in idx)

        def check(o):
            assert o == want

        t = timed(lambda: ctx.kzg_blob_to_commitment_and_cell_proofs(lag, mono, data), check, a.steps, a.warmup)
        emit("kzg_blob_to_commitment_and_cell_proofs", n, call_ms=t,
             kernel_ms=phase_split(lambda: check(ctx.kzg_blob_to_commitment_and_cell_proofs(lag, mono, data))))
    for h in (lag, mono):
        ctx.bases_free(h)
    ctx.close()


if __name__ == "__main__":
    main()
