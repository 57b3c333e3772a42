"""What the zero-knowledge tail costs: the synthetic Groth16 prove (SyntheticWrapCircuit, one GPU) through
b200zk_groth16_commit (unblinded, C = L + H) and through b200zk_groth16_prove (alpha / beta / delta terms and r, s
blinding), the two alternating step by step in one process, and the two assembly calls alone -- b200zk_groth16_fold
against b200zk_groth16_fold_zk over the same 768-byte block -- timed with CUDA events on the calling stream.
Prints one JSON line per domain, with the card's name and power limit.

    python tools/groth16_zk_latency.py [--log-n 20 24] [--steps 10] [--warmup 2]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import ethrex_b200 as eb  # noqa: E402
from ethrex_b200 import _ffi as F  # noqa: E402
from ethrex_b200.groth16 import SyntheticWrapCircuit, random_scalar  # noqa: E402


def gpu_identity(index: int = 0) -> dict:
    try:
        out = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30, check=True).stdout.strip()
        name, watts = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit_w": float(watts)}
    except Exception:
        return {"name": torch.cuda.get_device_name(index), "power_limit_w": None}


def stats(xs):
    return {"min": min(xs), "median": statistics.median(xs), "max": max(xs)}


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, nargs="+", default=[20, 24])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    ctx = eb.Context(0)
    ident = gpu_identity(0)
    for log_n in args.log_n:
        circ = SyntheticWrapCircuit(ctx, log_n, zk=True)
        seed = b"groth16-zk-latency"
        r, s = random_scalar(), random_scalar()
        commit = lambda: circ.prove_device(seed)  # noqa: E731
        prove = lambda: circ.prove_zk_device(seed, r=r, s=s)  # noqa: E731
        for _ in range(args.warmup):
            commit()
            prove()
        t_commit, t_prove = [], []
        for i in range(args.steps):  # alternate which one goes first
            pair = ((commit, t_commit), (prove, t_prove)) if i % 2 == 0 else ((prove, t_prove), (commit, t_commit))
            for fn, out in pair:
                out.append(timed(fn))
        assert prove() == prove(), "the same r, s must give the same proof"
        # the assembly step alone, over one block of partial sums
        w, a, b, c = circ.assign(seed)
        block = torch.zeros(96, dtype=torch.int64, device="cuda")
        ctx.groth16_commit_partial(circ.pk_struct(), w, a, b, c, block, F.G16_INPUTS_DEVICE)
        hd = circ.pk.handles
        zk = ctx.groth16_zk(hd["terms_g1"], hd["terms_g2"], r, s)
        for _ in range(args.warmup):
            ctx.groth16_fold(block, 1)
            ctx.groth16_fold_zk(zk, block, 1)
        f_plain, f_zk = [], []
        for _ in range(args.steps):
            f_plain.append(event_ms(lambda: ctx.groth16_fold(block, 1)))
            f_zk.append(event_ms(lambda: ctx.groth16_fold_zk(zk, block, 1)))
        circ.close()
        del w, a, b, c, block
        torch.cuda.empty_cache()
        line = {"log_n": log_n, "steps": args.steps, "warmup": args.warmup, "gpu": ident,
                "groth16_commit_ms": stats(t_commit), "groth16_prove_ms": stats(t_prove),
                "median_difference_ms": statistics.median(t_prove) - statistics.median(t_commit),
                "fold_ms": stats(f_plain), "fold_zk_ms": stats(f_zk),
                "fold_median_difference_ms": statistics.median(f_zk) - statistics.median(f_plain)}
        print(json.dumps(line), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
