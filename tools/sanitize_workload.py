"""Small end-to-end workload for compute-sanitizer (memcheck / racecheck / synccheck): every kernel family once."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "oracle"))
import numpy as np, torch
import ethrex_b200 as eb, pyref, cpu_oracle as orc

ctx = eb.Context(0)
k, d = pyref.chain_scalar(pyref.SEED_POINTS)
dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.int64).copy()).cuda()
n = 5000
pts, s = orc.g1_chain(n, k, d), orc.rand_fr(7, 0, n)
exp = orc.g1_msm(pts, s)
dp, ds = dev(pts), dev(s)
assert ctx.g1_msm_device(dp, ds, n) == exp                       # one-shot plain
ctx.set_msm_chunks(3); assert ctx.g1_msm_device(dp, ds, n) == exp; ctx.set_msm_chunks(0)   # pipelined
h = ctx.g1_bases_upload(pts, n); ctx.bases_precompute(h, 8)
assert ctx.g1_msm_resident(h, s, n) == exp                        # table + host scalars
ctx.bases_free(h)
p2 = orc.g2_chain(600, k, d)
assert ctx.g2_msm_device(dev(p2), dev(s[:600]), 600) == orc.g2_msm(p2, s[:600])
for log_n in (3, 9, 12, 14, 17):  # 17: the last pass's direct twiddle table (forward, inverse scaled, inverse unscaled)
    a = orc.fr_to_mont(orc.rand_fr(9, 0, 1 << log_n)); da = dev(a)
    ctx.fr_ntt_device(da, log_n, 0)
    assert (da.cpu().numpy().view(np.uint64).reshape(-1, 4) == orc.fr_ntt(a, log_n)).all()
    ctx.fr_ntt_device(da, log_n, eb.NTT_INVERSE)
    ctx.fr_ntt_device(da, log_n, eb.NTT_COSET)
    ctx.fr_ntt_device(da, log_n, eb.NTT_COSET | eb.NTT_INVERSE)
    assert (da.cpu().numpy().view(np.uint64).reshape(-1, 4) == a).all()
# ---- round 2: two-level sort (n >= 2^16), plain and table bases, host scalars through the one-stream pipeline
n2 = 70000
g2n = torch.empty(8 * n2, dtype=torch.int64, device="cuda"); ctx.g1_chain_device(g2n, 0, n2, k, d)
s2 = torch.empty(4 * n2, dtype=torch.int64, device="cuda"); ctx.fr_random_device(s2, n2, 77, 0)
ref2 = ctx.g1_msm_device(g2n, s2, n2)
import os as _os
h2 = ctx.g1_bases_from_device(g2n, n2); ctx.bases_precompute(h2, 0)
assert ctx.g1_msm_resident_device(h2, s2, n2) == ref2
ctx.set_msm_chunks(2); assert ctx.g1_msm_resident(h2, s2.cpu().numpy(), n2) == ref2; ctx.set_msm_chunks(0)
ctx.bases_free(h2)
exp2 = orc.g1_msm(g2n.cpu().numpy().view(np.uint64).reshape(n2, 8), s2.cpu().numpy().view(np.uint64).reshape(n2, 4))
assert ref2 == exp2
# ---- G2 on lane pairs over a window table; the one-call Groth16 path; NTT under halo2curves' root; BLS12-381
hg2 = ctx.g2_bases_upload(p2, 600); ctx.bases_precompute(hg2, 0)
assert ctx.g2_msm_resident(hg2, s[:600], 600) == orc.g2_msm(p2, s[:600]); ctx.bases_free(hg2)
from ethrex_b200.groth16 import SyntheticWrapCircuit
circ = SyntheticWrapCircuit(ctx, 8, precompute=True)
pr, b1 = circ.prove_device(b"sanitize"); pr2, cm = circ.prove_separate(b"sanitize"); assert pr == pr2 and b1 == cm["b_g1"]; circ.close()
ctx.set_ntt_root(ctx.ntt_root_preset(1)); a = orc.fr_to_mont(orc.rand_fr(9, 0, 1 << 10)); da = dev(a); ctx.fr_ntt_device(da, 10, 0)
assert (da.cpu().numpy().view(np.uint64).reshape(-1, 4) == orc.fr_ntt(a, 10, 0, root_2_28=pow(7, (pyref.R - 1) >> 28, pyref.R))).all(); ctx.set_ntt_root(None)
import bls_ref as bls
bp = bls.generator_multiples([3 + 5 * i for i in range(40)]); bs_ = [(i * 0x9E3779B97F4A7C15 + 1) % bls.R for i in range(40)]
hb = ctx.bls12_381_g1_bases_upload(b"".join(bls.compress(x) for x in bp), 40)
assert ctx.bls12_381_g1_msm_resident(hb, b"".join(v.to_bytes(32, "big") for v in bs_), 40) == bls.compress(bls.msm(bs_, bp)); ctx.bases_free(hb)
g = torch.empty(8 * 300, dtype=torch.int64, device="cuda"); ctx.g1_chain_device(g, 0, 300, k, d); assert ctx.g1_check_device(g, 300) == 300
print("sanitize workload ok, launches:", ctx.launch_count)
ctx.close()
