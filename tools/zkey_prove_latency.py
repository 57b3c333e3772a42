"""Latency of Groth16 from circom artifacts (b200zk_groth16_zkey_load / _prove) at domain 2^22 and 2^23, next to the
existing one-call prove (b200zk_groth16_prove over the synthetic ark-layout key) at the same domain, in the same run.

The .zkey is assembled in memory: its points come from b200zk_g1/g2_chain_device (whose output is the zkey's native
layout already), its section-4 rows are random with a skewed length distribution (most rows 1-8 terms, every 4096th row
2048 terms), and the witness is random.  The prover does not check that the rows are satisfied, so the work is what a
real circuit of this shape costs.  Prints the card's name and power limit, then one JSON line per domain: load and prove
wall-clock medians, and the device time of a prove split into evaluation, NTTs + quotient, MSMs, assembly,
copies and other kernels (median over `steps` profiled proves, each profiled on its own).

    python tools/zkey_prove_latency.py [--log-n 22 23] [--steps 5] [--warmup 1]
"""
from __future__ import annotations

import argparse
import json
import os
import struct
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

R = 0x30644E72E131A029B85045B68181585D2833E84879B9709143E1F593F0000001
Q = 0x30644E72E131A029B85045B68181585D97816A916871CA8D3C208C16D87CFD47


def _chain(ctx, g2: bool, n: int, k: int) -> bytes:
    import torch
    pts = torch.empty((16 if g2 else 8) * n, dtype=torch.int64, device="cuda")
    (ctx.g2_chain_device if g2 else ctx.g1_chain_device)(pts, 0, n, k, 2 * k + 1)
    return pts.cpu().numpy().tobytes()


def _random_fr(rng, n: int) -> np.ndarray:
    """n values < r as 8 little-endian u32 limbs (top limb below r's)"""
    v = rng.integers(0, 1 << 32, size=(n, 8), dtype=np.uint64).astype(np.uint32)
    v[:, 7] %= 0x30644E72
    return v


def build_files(ctx, log_n: int, seed: int = 1):
    rng = np.random.default_rng(seed)
    n = 1 << log_n
    n_public, n_vars = 2, n - 8
    rows = n - n_public - 1
    rec_dtype = np.dtype([("m", "<u4"), ("c", "<u4"), ("s", "<u4"), ("v", "<u4", (8,))])
    parts = []
    for m in (0, 1):
        lens = np.minimum(rng.geometric(0.45, size=rows), 8).astype(np.int64)
        lens[::4096] = 2048
        cons = np.repeat(np.arange(rows, dtype=np.uint32), lens)
        rec = np.empty(len(cons), dtype=rec_dtype)
        rec["m"], rec["c"] = m, cons
        rec["s"] = rng.integers(0, n_vars, size=len(cons), dtype=np.uint32)
        rec["v"] = _random_fr(rng, len(cons))
        parts.append(rec)
    pad = np.empty(n_public + 1, dtype=rec_dtype)
    pad["m"], pad["c"], pad["s"] = 0, rows + np.arange(n_public + 1), np.arange(n_public + 1)
    pad["v"] = 0
    pad["v"][:, 0] = 1
    recs = np.concatenate(parts + [pad])
    recs = recs[rng.permutation(len(recs))]
    g1, g2 = _chain(ctx, False, 6, 101), _chain(ctx, True, 3, 103)
    hdr = struct.pack("<I", 32) + Q.to_bytes(32, "little") + struct.pack("<I", 32) + R.to_bytes(32, "little") + struct.pack("<III", n_vars, n_public, n)
    hdr += g1[0:64] + g1[64:128] + g2[0:128] + g2[128:256] + g1[128:192] + g2[256:384]

    def sec(i, payload):
        return struct.pack("<IQ", i, len(payload)), payload

    pieces = [b"zkey", struct.pack("<II", 1, 9)]
    for i, payload in ((1, struct.pack("<I", 1)), (2, hdr), (3, g1[:64 * (n_public + 1)]), (4, struct.pack("<I", len(recs)) + recs.tobytes()),
                       (5, _chain(ctx, False, n_vars, 3)), (6, _chain(ctx, False, n_vars, 5)), (7, _chain(ctx, True, n_vars, 7)),
                       (8, _chain(ctx, False, n_vars - n_public - 1, 11)), (9, _chain(ctx, False, n, 13))):
        pieces += sec(i, payload)
    zkey = b"".join(pieces)
    wit = _random_fr(rng, n_vars)
    wit[0] = 0
    wit[0, 0] = 1
    body = wit.tobytes()
    wtns = b"wtns" + struct.pack("<II", 2, 2) + struct.pack("<IQ", 1, 40) + struct.pack("<I", 32) + R.to_bytes(32, "little") + struct.pack("<I", n_vars)
    wtns += struct.pack("<IQ", 2, len(body)) + body
    return zkey, wtns, len(recs)


# kernel families of a zkey prove, by name prefix; anything else is reported as "other", never folded into a phase
PHASES = (("evaluation", ("zkey_eval", "zkey_wtns", "field_mul_kernel")),
          ("ntt_quotient", ("ntt_", "fr_quotient")),
          ("msm", ("msm_", "bucket_", "partial_tree", "scan_", "write_identity")),
          ("assembly", ("groth16_assemble",)),
          ("copies", ("Memcpy", "Memset", "memcpy", "memset")))


def _phase(name: str) -> str:
    for phase, keys in PHASES:
        if any(k in name for k in keys):
            return phase
    return "other"


def profile_phases(fn, calls: int) -> dict:
    """device time (ms) of `calls` profiled calls, by kernel family: the median over the calls of each family's total"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    per_call = []
    for _ in range(calls):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        out = dict.fromkeys([p for p, _ in PHASES] + ["other"], 0.0)
        for ev in prof.key_averages():
            t = getattr(ev, "device_time_total", None)
            if t is None:
                t = ev.cuda_time_total
            if t > 0:
                out[_phase(ev.key)] += t / 1000
        per_call.append(out)
    return {k: round(float(np.median([c[k] for c in per_call])), 3) for k in per_call[0]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, nargs="+", default=[22, 23])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    import torch
    import ethrex_b200 as eb
    from ethrex_b200.groth16 import SyntheticWrapCircuit
    from ethrex_b200.zkey import ZkeyProver
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement needs the GPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"card: {card}", flush=True)
    ctx = eb.Context(0)
    r, s = 0x1234567 << 100, 0x7654321 << 90
    for log_n in args.log_n:
        zkey, wtns, nnz = build_files(ctx, log_n)
        loads = []
        for i in range(args.warmup + args.steps):
            t0 = time.perf_counter()
            p = ZkeyProver(ctx, zkey, precompute=True)
            dt = time.perf_counter() - t0
            if i >= args.warmup:
                loads.append(dt)
            if i < args.warmup + args.steps - 1:
                p.close()
        del zkey
        proves = []
        for i in range(args.warmup + args.steps):
            t0 = time.perf_counter()
            proof = p.prove(wtns, r=r, s=s)
            dt = time.perf_counter() - t0
            if i >= args.warmup:
                proves.append(dt)
        assert p.prove(wtns, r=r, s=s) == proof  # reproducible
        phases = profile_phases(lambda: p.prove(wtns, r=r, s=s), args.steps)
        p.close()
        torch.cuda.empty_cache()
        circ = SyntheticWrapCircuit(ctx, log_n, precompute=True, zk=True)
        base = []
        for i in range(args.warmup + args.steps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            circ.prove_zk_device(b"zkey-latency", r=r, s=s)
            dt = time.perf_counter() - t0
            if i >= args.warmup:
                base.append(dt)
        circ.close()
        torch.cuda.empty_cache()
        res = {"log_n": log_n, "nnz": nnz, "wtns_bytes": len(wtns), "zkey_load_ms": round(1e3 * float(np.median(loads)), 2),
               "zkey_prove_ms": round(1e3 * float(np.median(proves)), 2), "zkey_prove_device_ms": phases,
               "groth16_prove_ms": round(1e3 * float(np.median(base)), 2), "steps": args.steps, "warmup": args.warmup, "card": card}
        print(json.dumps(res), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
