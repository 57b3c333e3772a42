"""Latency and memory of b200zk_plonk_zkey_prove at circuit sizes, with the Groth16 zkey prove at the same domain.

    python tools/plonk_prove_latency.py --log-n 20 22 --reps 3

For each log_n: a snarkjs 0.7 PLONK key of tests/plonk_ref.py (its polynomial sections from the C++ oracle's NTTs, PTau
from the device's batched scalar multiplication), loaded with window tables, then
  - the median of `--reps` proves, timed with CUDA events around the one C-ABI call, the proof checked by PlonkVerifier;
  - the per-round split of one more prove with profiling on (b200zk_plonk_last_round_ms: CUDA events at the round
    boundaries; profiling runs the MSMs unchunked, so its total may differ a little from the median);
  - device memory in use after load and after the first prove (cudaMemGetInfo).  The library's workspaces only grow and a
    prove frees nothing, so the usage after the first prove is the prove's peak; load may hold PTau twice for a moment
    while the window table is built (+64 (n + 6) bytes).  Printed next to the figures derived from the carve sizes
    (DESIGN.md section 4.18) and the largest log_n that derivation fits into this card's memory;
  - the Groth16 zkey prove (tools/zkey_prove_latency.py's files at the same domain), median of `--reps`.
`--chain L` adds a 2^16 key whose additions form one chain of L levels next to one with the same additions unchained.
The card's name and power limit are printed with the numbers."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tools")):
    sys.path.insert(0, p)

import torch  # noqa: E402

import ethrex_b200 as eb  # noqa: E402
import plonk_ref as pr  # noqa: E402
from ethrex_b200 import _ffi as F  # noqa: E402
from ethrex_b200.zkey import PlonkProver, ZkeyProver  # noqa: E402
from zkey_prove_latency import build_files  # noqa: E402

ROUNDS = ("round1_wires", "round2_z", "round3_quotient", "round4_evals", "round5_openings")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def key_bytes(n: int, table_windows: int) -> int:
    """DESIGN 4.18: 8n coefficients + 9 x 4n coset values + 3n domain values (32 B each) + PTau with its window table"""
    return 47 * n * 32 + 64 * (n + 6) * table_windows


def workspace_bytes(n: int, n_vars: int, n_public: int) -> int:
    """DESIGN 4.18, the carve of plonk.cu's prove(): the witness, 3n + 4(n+8) + 20n + 4n + 3(n+8) + n + 2(n+8) values, the
    scan state (3 values per 32-element chunk) and small blocks"""
    chunks = (n + 8 + 31) // 32
    return 32 * (n_vars + 37 * n + 72 + 3 * chunks + 1) + 32 * n_public + 64 * 1024


def timed(fn, reps):
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return times


def used():
    torch.cuda.synchronize()
    free, total = torch.cuda.mem_get_info()
    return total - free, total


def plonk_case(ctx, log_n, reps, chain=0.5, n_additions=None):
    n = 1 << log_n
    t0 = time.time()
    c = pr.PlonkCircuit(n_gates=n - n // 8, n_public=2, n_private=64, n_additions=n // 16 if n_additions is None else n_additions,
                        seed=log_n, log_n=log_n, chain=chain)
    zkey = c.zkey(ctx)
    wt = c.assign([3, 4])
    wtns, pub = c.wtns(wt), c.public(wt)
    fixture_s = time.time() - t0
    u0, total = used()
    t0 = time.time()
    prover = PlonkProver(ctx, zkey, precompute=True)
    load_s = time.time() - t0
    u1, _ = used()
    blinding = [7 + k for k in range(11)]
    proof = prover.prove(wtns, blinding)
    u2, _ = used()
    assert prover.verifier().verify(proof, pub), "the proof does not verify"
    times = timed(lambda: prover.prove(wtns, blinding), reps)
    ctx.set_profiling(True)
    prover.prove(wtns, blinding)
    rounds = (C.c_float * 5)()
    ctx._check(F.lib.b200zk_plonk_last_round_ms(ctx._h, rounds), "b200zk_plonk_last_round_ms")
    ctx.set_profiling(False)
    prover.close()
    levels = 0
    if c.adds:
        lv = []
        for s1, s2, _, _ in c.adds:
            lv.append(1 + max([lv[s - c.n_wtns] for s in (s1, s2) if s >= c.n_wtns] or [0]))
        levels = max(lv)
    return {"log_n": log_n, "prove_ms_median": round(statistics.median(times), 2), "prove_ms": [round(t, 2) for t in times],
            "rounds_ms": {k: round(v, 2) for k, v in zip(ROUNDS, rounds)}, "verified": True, "load_s": round(load_s, 2),
            "key_mib": round((u1 - u0) / 2**20, 1), "prove_workspace_mib": round((u2 - u1) / 2**20, 1),
            "n_additions": c.n_additions, "addition_levels": levels, "fixture_s": round(fixture_s, 1), "n_vars": c.n_vars, "total_mib": total >> 20}


def groth16_case(ctx, log_n, reps):
    zkey, wtns, _ = build_files(ctx, log_n)
    prover = ZkeyProver(ctx, zkey, precompute=True)
    prover.prove(wtns, r=5, s=7)
    times = timed(lambda: prover.prove(wtns, r=5, s=7), reps)
    prover.close()
    return {"log_n": log_n, "groth16_zkey_prove_ms_median": round(statistics.median(times), 2), "prove_ms": [round(t, 2) for t in times]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, nargs="+", default=[20, 22])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--chain", type=int, default=0, help="length of one addition chain to time at 2^16 (0: skip)")
    ap.add_argument("--no-groth16", action="store_true")
    args = ap.parse_args()
    print("card:", card(), flush=True)
    ctx = eb.Context(0)
    for log_n in args.log_n:
        r = plonk_case(ctx, log_n, args.reps)
        n = 1 << log_n
        tw = (255 + 19) // 20 if log_n >= 20 else None
        if tw:
            r["derived_key_mib"] = round(key_bytes(n, tw) / 2**20, 1)
        r["derived_workspace_mib"] = round(workspace_bytes(n, r["n_vars"], 2) / 2**20, 1)
        print(json.dumps({"plonk": r}), flush=True)
        if not args.no_groth16:
            print(json.dumps({"groth16_zkey": groth16_case(ctx, log_n, args.reps)}), flush=True)
        total = r["total_mib"] << 20
        fits = max(lg for lg in range(10, 27) if key_bytes(1 << lg, 13) + workspace_bytes(1 << lg, 1 << lg, 2) <= total)
        print(json.dumps({"largest_log_n_by_derivation": fits, "card_mib": r["total_mib"]}), flush=True)
    if args.chain:
        flat = plonk_case(ctx, 16, args.reps, chain=0.0, n_additions=args.chain)
        chained = plonk_case(ctx, 16, args.reps, chain=1.0, n_additions=args.chain)
        print(json.dumps({"additions": args.chain, "levels_unchained": flat["addition_levels"], "prove_ms_unchained": flat["prove_ms_median"],
                          "levels_chained": chained["addition_levels"], "prove_ms_chained": chained["prove_ms_median"]}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
