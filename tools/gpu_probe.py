"""Exploration probe (not the bench): times the field core, the NTT and MSM windows on one GPU and
writes JSON lines to gpurun_out/probe.jsonl.  Usage: python tools/gpu_probe.py [section ...]"""
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import ethrex_b200 as eb  # noqa: E402

OUT = os.path.join(ROOT, "gpurun_out")
os.makedirs(OUT, exist_ok=True)
LOG = open(os.path.join(OUT, "probe.jsonl"), "a")


def emit(**kw):
    line = json.dumps(kw)
    print(line, flush=True)
    LOG.write(line + "\n")
    LOG.flush()


def timed(fn, iters=5, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2], ts[0]


def dev(n_u64):
    return torch.empty(n_u64, dtype=torch.int64, device="cuda")


def main():
    sections = sys.argv[1:] or ["field", "ntt", "msm"]
    ctx = eb.Context(0)
    emit(section="env", gpu=torch.cuda.get_device_name(0), sms=torch.cuda.get_device_properties(0).multi_processor_count)
    if "field" in sections:
        n = 1 << 22
        a, b, o = dev(4 * n), dev(4 * n), dev(4 * n)
        ctx.fr_random_device(a, n, 1, 0)
        ctx.fr_random_device(b, n, 2, 0)
        for which in (0, 1):
            for rep in (64, 256):
                med, best = timed(lambda: ctx.field_mul_device(a, b, o, n, which, rep), iters=5)
                emit(section="field", which=which, n=n, repeat=rep, ms=med, gmul_per_s=n * rep / best / 1e6)
    if "ntt" in sections:
        for log_n in (20, 24):
            n = 1 << log_n
            d = dev(4 * n)
            ctx.fr_random_device(d, n, 3, 0, eb.SCALARS_MONT)
            try:
                med, best = timed(lambda: ctx.fr_ntt_device(d, log_n, 0), iters=5)
                emit(section="ntt", log_n=log_n, ms=med, best_ms=best, gelem_per_s=n / best / 1e6)
            except Exception as e:  # noqa: BLE001
                emit(section="ntt", log_n=log_n, error=str(e))
    if "msm" in sections:
        import pyref
        k, dd = pyref.chain_scalar(pyref.SEED_POINTS)
        for log_n, windows in ((20, (0,)), (24, (0,))):
            n = 1 << log_n
            p, s = dev(8 * n), dev(4 * n)
            t0 = time.time()
            ctx.g1_chain_device(p, 0, n, k, dd)
            ctx.synchronize()
            emit(section="chain", log_n=log_n, seconds=time.time() - t0)
            ctx.fr_random_device(s, n, pyref.SEED_SCALARS, 0)
            ctx.set_profiling(True)
            for c in windows:
                ctx.set_msm_window(c)
                try:
                    med, best = timed(lambda: ctx.g1_msm_device(p, s, n), iters=3, warm=1)
                    emit(section="msm_g1", log_n=log_n, c=c, ms=med, best_ms=best, mpts_per_s=n / best / 1e3, phases=ctx.last_msm_phase_ms())
                except Exception as e:  # noqa: BLE001
                    emit(section="msm_g1", log_n=log_n, c=c, error=str(e))
            ctx.set_msm_window(0)
            ctx.set_profiling(False)
        # precomputed window tables
        for log_n, windows in ((16, (0,)), (20, (0,)), (24, (0,))):
            n = 1 << log_n
            p, s = dev(8 * n), dev(4 * n)
            ctx.g1_chain_device(p, 0, n, k, dd)
            ctx.fr_random_device(s, n, pyref.SEED_SCALARS, 0)
            ctx.set_profiling(True)
            for c in windows:
                try:
                    t0 = time.time()
                    h = ctx.g1_bases_from_device(p, n)
                    ctx.bases_precompute(h, c)
                    ctx.synchronize()
                    build_s = time.time() - t0
                    med, best = timed(lambda: ctx.g1_msm_resident_device(h, s, n), iters=3, warm=1)
                    emit(section="msm_g1_pre", log_n=log_n, c=c, build_s=build_s, ms=med, best_ms=best, mpts_per_s=n / best / 1e3, phases=ctx.last_msm_phase_ms())
                    ctx.bases_free(h)
                except Exception as e:  # noqa: BLE001
                    emit(section="msm_g1_pre", log_n=log_n, c=c, error=str(e))
            ctx.set_profiling(False)
            del p, s
        n = 1 << 20
        p, s = dev(16 * n), dev(4 * n)
        ctx.g2_chain_device(p, 0, n, k, dd)
        ctx.fr_random_device(s, n, pyref.SEED_SCALARS, 0)
        ctx.set_profiling(True)
        med, best = timed(lambda: ctx.g2_msm_device(p, s, n), iters=3, warm=1)
        emit(section="msm_g2", log_n=20, ms=med, best_ms=best, mpts_per_s=n / best / 1e3, phases=ctx.last_msm_phase_ms())
    ctx.close()


if __name__ == "__main__":
    main()
