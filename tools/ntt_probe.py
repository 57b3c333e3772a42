import os, sys, json, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "oracle"))
import ethrex_b200 as eb, pyref
ctx = eb.Context(0)
def timed(fn, iters=7, warm=3):
    for _ in range(warm): fn()
    torch.cuda.synchronize(); ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize(); ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]
for log_n in (20, 22, 24):
    n = 1 << log_n
    d = torch.empty(4 * n, dtype=torch.int64, device="cuda")
    ctx.fr_random_device(d, n, 3, 0, eb.SCALARS_MONT)
    for flags, name in ((0, "fwd"), (eb.NTT_INVERSE, "inv"), (eb.NTT_COSET, "coset"), (eb.NTT_COSET | eb.NTT_INVERSE, "coset_inv")):
        ms = timed(lambda: ctx.fr_ntt_device(d, log_n, flags))
        print(json.dumps({"log_n": log_n, "mode": name, "ms": round(ms, 4), "gelem_s": round(n / ms / 1e6, 3)}), flush=True)
