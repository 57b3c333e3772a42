"""GPU parity tests added in round 2: the configurations BASELINE.json names at their full sizes (G2 MSM at 2^22 / 2^24,
the sharded G1+G2 MSM of config 4), the NTT root-of-unity parameter (halo2curves' root for the OpenVM wrap), the
one-call Groth16 entry point against the separate-call pipeline, the ABI v2 asynchronous forms, and the verifier's
canonical-encoding rules.  Same shape as tests/test_gpu_parity.py: bytes in, bytes out, compared with the CPU oracle
or with a closed form the oracle evaluates."""
import os
import subprocess
import sys

import numpy as np
import pytest

import cpu_oracle as orc
import pyref
from helpers import chain_kd, dev_empty, expected_chain_msm_g1, expected_chain_msm_g2, to_dev, to_host

pytestmark = pytest.mark.gpu

import ethrex_b200 as eb  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HALO2_ROOT = pow(7, (pyref.R - 1) >> 28, pyref.R)
ARK_ROOT = pow(5, (pyref.R - 1) >> 28, pyref.R)


# ------------------------------------------------------------------------------------------ config 4 sizes, one GPU
@pytest.mark.parametrize("log_n,table", [(22, False), (22, True), (24, True)])
def test_g2_msm_large_closed_form(ctx, log_n, table):
    """G2 MSM at 2^22 (plain and window-table bases) and 2^24 (tables: the configuration the bench times): the chain
    bases make the exact answer one scalar multiplication of the EIP-197 generator."""
    import torch
    n = 1 << log_n
    k, d = chain_kd()
    dp, ds = dev_empty(16 * n), dev_empty(4 * n)
    ctx.g2_chain_device(dp, 0, n, k, d)
    ctx.fr_random_device(ds, n, pyref.SEED_SCALARS, 0)
    exp = expected_chain_msm_g2(to_host(ds).reshape(n, 4), k, d)
    if table:
        h = ctx.g2_bases_from_device(dp, n)
        del dp
        torch.cuda.empty_cache()
        try:
            ctx.bases_precompute(h, 0)
            assert ctx.g2_msm_resident_device(h, ds, n) == exp
        finally:
            ctx.bases_free(h)
    else:
        assert ctx.g2_check_device(dp, n) == n
        assert ctx.g2_msm_device(dp, ds, n) == exp
    torch.cuda.empty_cache()


def test_g1_g2_msm_point_split_equals_whole_at_2_22(ctx):
    """config 4's partitioning on one device: a 2^22-point MSM cut into 8 point shards, each reduced to an XYZZ partial,
    folded -- equal to the unsharded call and to the closed form, for G1 and G2 (the N-GPU run moves the same partials
    through one all_gather: tests/test_gpu_r2.py::test_sharded_g1_g2_msm_two_ranks, bench.py `strong`)."""
    import torch
    n, parts = 1 << 22, 8
    k, d = chain_kd()
    ds = dev_empty(4 * n)
    ctx.fr_random_device(ds, n, pyref.SEED_SCALARS, 0)
    s = to_host(ds).reshape(n, 4)
    for g2 in (False, True):
        w = 16 if g2 else 8
        dp = dev_empty(w * n)
        (ctx.g2_chain_device if g2 else ctx.g1_chain_device)(dp, 0, n, k, d)
        partials = torch.zeros((32 if g2 else 16) * parts, dtype=torch.int64, device="cuda")
        step = n // parts
        for r in range(parts):
            fn = ctx.g2_msm_partial_device if g2 else ctx.g1_msm_partial_device
            fn(dp[w * r * step: w * (r + 1) * step], ds[4 * r * step: 4 * (r + 1) * step], step, partials[(32 if g2 else 16) * r:])
        got = (ctx.g2_fold_partials_device if g2 else ctx.g1_fold_partials_device)(partials, parts)
        exp = (expected_chain_msm_g2 if g2 else expected_chain_msm_g1)(s, k, d)
        assert got == exp
        assert (ctx.g2_msm_device if g2 else ctx.g1_msm_device)(dp, ds, n) == exp
        del dp
        torch.cuda.empty_cache()


def test_sharded_g1_g2_msm_two_ranks():
    """config 4 across processes: torchrun world 2 over NCCL, G1 and G2, 2^20 points in total, every rank must return
    the closed form (skipped on a one-GPU box; bench.py --gpus N runs the same path at 2^24)."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    script = os.path.join(ROOT, "tests", "sharded_worker.py")
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                        "--master-port", "29617", script, "20"], capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert r.stdout.count("SHARDED_OK") == 2


# ------------------------------------------------------------------------------------------ NTT root parameter
def test_ntt_root_presets_are_the_published_generators(ctx):
    assert int.from_bytes(ctx.ntt_root_preset(0), "little") == ARK_ROOT
    assert int.from_bytes(ctx.ntt_root_preset(1), "little") == HALO2_ROOT == 0x03ddb9f5166d18b798865ea93dd31f743215cf6dd39329c8d34f1ed960c37c9c
    with pytest.raises(eb.B200Error):
        ctx.ntt_root_preset(2)


@pytest.mark.parametrize("log_n", [1, 5, 12, 16, 20])
def test_ntt_with_halo2curves_root_matches_oracle(ctx, log_n):
    """SURVEY.md section 8c: halo2curves derives its domains from 7^((r-1)/2^28), not ark/gnark's 5^((r-1)/2^28); with
    the context switched to that root every mode must equal the oracle run with the same root -- and differ from the
    default-root transform -- and switching back must restore the default bit for bit."""
    n = 1 << log_n
    a = orc.fr_to_mont(orc.rand_fr(pyref.SEED_NTT, 0, n))
    default_fwd = orc.fr_ntt(a, log_n, 0)
    try:
        ctx.set_ntt_root(ctx.ntt_root_preset(1))
        for flags_gpu, flags_orc in ((0, 0), (eb.NTT_INVERSE, orc.NTT_INVERSE), (eb.NTT_COSET, orc.NTT_COSET), (eb.NTT_INVERSE | eb.NTT_COSET, orc.NTT_INVERSE | orc.NTT_COSET)):
            d = to_dev(a)
            ctx.fr_ntt_device(d, log_n, flags_gpu)
            exp = orc.fr_ntt(a, log_n, flags_orc, root_2_28=HALO2_ROOT)
            assert (to_host(d).reshape(n, 4) == exp).all(), (log_n, flags_gpu)
        # the two generators are powers of each other (7^t = (5^t)^x): their 2^k-th roots coincide while x = 1 mod 2^k, which
        # happens to hold for small k -- so "differs from the default" is asserted exactly when the oracle says so
        halo2_fwd = orc.fr_ntt(a, log_n, 0, root_2_28=HALO2_ROOT)
        d = to_dev(a)
        ctx.fr_ntt_device(d, log_n, 0)
        assert bool((to_host(d).reshape(n, 4) == default_fwd).all()) == bool((halo2_fwd == default_fwd).all())
        if log_n >= 12:
            assert not (halo2_fwd == default_fwd).all()
    finally:
        ctx.set_ntt_root(None)
    d = to_dev(a)
    ctx.fr_ntt_device(d, log_n, 0)
    assert (to_host(d).reshape(n, 4) == default_fwd).all()


def test_ntt_root_must_be_a_primitive_2_28th_root(ctx):
    for bad in (1, pyref.R - 1, pow(ARK_ROOT, 2, pyref.R), 5, pyref.R + ARK_ROOT):  # order 1, 2, 2^27, not a root, not canonical
        with pytest.raises(eb.B200Error):
            ctx.set_ntt_root((bad % (1 << 256)).to_bytes(32, "little"))
    # a rejected root leaves the context on its previous one
    a = orc.fr_to_mont(orc.rand_fr(pyref.SEED_NTT, 0, 16))
    d = to_dev(a)
    ctx.fr_ntt_device(d, 4, 0)
    assert (to_host(d).reshape(16, 4) == orc.fr_ntt(a, 4, 0)).all()
    # any odd power of the generator is again primitive
    g3 = pow(ARK_ROOT, 3, pyref.R)
    try:
        ctx.set_ntt_root(g3.to_bytes(32, "little"))
        d = to_dev(a)
        ctx.fr_ntt_device(d, 4, 0)
        assert (to_host(d).reshape(16, 4) == orc.fr_ntt(a, 4, 0, root_2_28=g3)).all()
    finally:
        ctx.set_ntt_root(None)


def test_kzg_commit_flow_in_lagrange_basis_with_halo2_root(ctx):
    """The OpenVM wrap's commitment (halo2 KZG, /root/reference/crates/prover/src/backend/openvm.rs:52-56): a polynomial
    given by its evaluations on halo2curves' domain is committed against the Lagrange-basis SRS with ONE MSM; the same
    polynomial taken to coefficients (iNTT under halo2's root) and committed against the monomial SRS must give the same
    group element, and both must equal p(tau) * G.  The SRS is synthetic (known tau), as in tests/groth16_toy.py."""
    log_n, n = 8, 1 << 8
    tau = 0x1F2E3D4C5B6A79880123456789ABCDEF % pyref.R
    w = pow(HALO2_ROOT, 1 << (28 - log_n), pyref.R)
    evals = orc.array_to_ints(orc.rand_fr(0xB2004B5A, 0, n))
    # monomial SRS tau^i G and Lagrange SRS L_i(tau) G, L_i(tau) = w^i (tau^n - 1) / (n (tau - w^i))
    mono = [pow(tau, i, pyref.R) for i in range(n)]
    zt, ninv = (pow(tau, n, pyref.R) - 1) % pyref.R, pow(n, -1, pyref.R)
    lag = [pow(w, i, pyref.R) * zt % pyref.R * ninv % pyref.R * pow((tau - pow(w, i, pyref.R)) % pyref.R, -1, pyref.R) % pyref.R for i in range(n)]
    gen = pyref.g1_to_be(pyref.G1_GEN)
    srs = lambda ks: b"".join(orc.g1_mul_be(gen, k.to_bytes(32, "big"))[1] for k in ks)  # noqa: E731
    p_tau = sum(e * l for e, l in zip(evals, lag)) % pyref.R
    want = orc.g1_mul_be(gen, p_tau.to_bytes(32, "big"))[1]
    h_lag, h_mono = ctx.g1_bases_upload(srs(lag), n, eb.POINTS_BE), ctx.g1_bases_upload(srs(mono), n, eb.POINTS_BE)
    try:
        ev = to_dev(orc.ints_to_array(evals))
        assert ctx.g1_msm_resident_device(h_lag, ev, n) == want
        ctx.set_ntt_root(ctx.ntt_root_preset(1))
        ctx.field_to_mont_device(ev, n, 1)
        ctx.fr_ntt_device(ev, log_n, eb.NTT_INVERSE)  # evaluations on halo2's domain -> coefficients
        assert ctx.g1_msm_resident_device(h_mono, ev, n, eb.SCALARS_MONT) == want
        # under the DEFAULT root the same evaluations describe another polynomial: the commitment must differ
        ctx.set_ntt_root(None)
        ev2 = to_dev(orc.fr_to_mont(orc.ints_to_array(evals)))
        ctx.fr_ntt_device(ev2, log_n, eb.NTT_INVERSE)
        assert ctx.g1_msm_resident_device(h_mono, ev2, n, eb.SCALARS_MONT) != want
    finally:
        ctx.set_ntt_root(None)
        ctx.bases_free(h_lag)
        ctx.bases_free(h_mono)


# ------------------------------------------------------------------------------------------ ABI v2
def test_async_msm_forms_append_the_infinity_word(ctx):
    import torch
    n = 64
    k, d = chain_kd()
    for g2 in (False, True):
        pts = (orc.g2_chain if g2 else orc.g1_chain)(n, k, d)
        s = orc.rand_fr(pyref.SEED_SCALARS, 0, n)
        size = 128 if g2 else 64
        out = torch.full((size // 8 + 1,), -1, dtype=torch.int64, device="cuda")
        fn = ctx.g2_msm_device_async if g2 else ctx.g1_msm_device_async
        fn(to_dev(pts), to_dev(s), n, out)
        raw = out.cpu().numpy().tobytes()
        assert raw[:size] == (orc.g2_msm if g2 else orc.g1_msm)(pts, s)
        assert raw[size:size + 4] == b"\0\0\0\0" and raw[size + 4:size + 8] == b"\xff\xff\xff\xff"  # flag written, nothing behind it
        fn(to_dev(pts), to_dev(np.zeros((n, 4), dtype=np.uint64)), n, out)  # all-zero scalars: the identity
        raw = out.cpu().numpy().tobytes()
        assert raw[:size] == bytes(size) and raw[size:size + 4] == b"\x01\0\0\0"
        with pytest.raises(eb.B200Error):
            fn(to_dev(pts), to_dev(s), n, torch.zeros(size // 8, dtype=torch.int64, device="cuda"))  # no room for the flag


def test_host_entry_points_refuse_short_buffers(ctx):
    """ADVICE r1: a short Python buffer must raise, not be read past its end."""
    pts, sc = bytes(64 * 4), bytes(32 * 4)
    with pytest.raises(eb.B200Error, match="needs"):
        ctx.g1_msm(pts, sc, 5, eb.POINTS_BE)
    with pytest.raises(eb.B200Error, match="needs"):
        ctx.g2_msm(bytes(128 * 2), sc, 3, eb.POINTS_BE)
    with pytest.raises(eb.B200Error, match="needs"):
        ctx.fr_ntt(bytearray(32 * 7), 3)
    with pytest.raises(eb.B200Error, match="needs"):
        ctx.g1_bases_upload(pts, 5, eb.POINTS_BE)
    h = ctx.g1_bases_upload(pts, 4, eb.POINTS_BE)
    try:
        with pytest.raises(eb.B200Error, match="needs"):
            ctx.g1_msm_resident(h, sc, 5)
        assert ctx.g1_msm_resident(h, sc, 4) == bytes(64)
    finally:
        ctx.bases_free(h)


def test_two_contexts_and_a_foreign_current_device(ctx):
    """ADVICE r1: every entry point runs on its context's device whatever torch's current device is.  On a one-GPU box
    this exercises the guard's no-op path with two contexts alive; with two GPUs the second context lives on cuda:1
    while torch's current device stays cuda:0."""
    import torch
    dev = 1 if torch.cuda.device_count() > 1 else 0
    other = eb.Context(dev)
    try:
        n = 256
        k, d = chain_kd()
        pts, s = orc.g1_chain(n, k, d), orc.rand_fr(pyref.SEED_SCALARS, 0, n)
        exp = orc.g1_msm(pts, s)
        be = orc.g1_native_to_be(pts)
        assert torch.cuda.current_device() == 0
        assert other.g1_msm(be, s, n, eb.POINTS_BE) == exp          # host entry point on the other context
        assert ctx.g1_msm(be, s, n, eb.POINTS_BE) == exp
        a = orc.fr_to_mont(orc.rand_fr(pyref.SEED_NTT, 0, 1 << 10))
        buf = bytearray(a.tobytes())
        other.fr_ntt(buf, 10)
        assert bytes(buf) == orc.fr_ntt(a, 10).tobytes()
        assert torch.cuda.current_device() == 0                      # the caller's device is restored
    finally:
        other.close()
    assert torch.cuda.current_device() == 0


# ------------------------------------------------------------------------------------------ Groth16: one call
@pytest.mark.parametrize("log_n,precompute", [(6, False), (10, True), (14, True)])
def test_groth16_one_call_equals_separate_calls(ctx, log_n, precompute):
    """b200zk_groth16_commit (device inputs, shared sort, on-device C = L + H, one read-back) against the same pipeline
    sequenced call by call from Python -- same proof bytes, and [B]1 equal to the separately computed commitment."""
    from ethrex_b200.groth16 import SyntheticWrapCircuit
    circuit = SyntheticWrapCircuit(ctx, log_n, precompute=precompute)
    try:
        for inp in (b"batch-1", b"batch-2"):
            proof, b1 = circuit.prove_device(inp)
            proof2, cm = circuit.prove_separate(inp)
            assert proof == proof2
            assert b1 == cm["b_g1"]
        # point split on ONE device: three "ranks" commit disjoint scalar ranges (the rest zeroed: zero digits add
        # nothing) into three 768-byte blocks; folding them must give the whole proof -- what N ranks all_gather
        import torch
        from ethrex_b200 import _ffi as F
        n = 1 << log_n
        whole, b1_whole = circuit.prove_device(b"batch-3")
        w, a, b, c = circuit.assign(b"batch-3")
        h = circuit.quotient(a, b, c)
        blocks = torch.zeros(96 * 3, dtype=torch.int64, device="cuda")
        hd = circuit.pk.handles
        pk = ctx.groth16_pk(log_n, [hd["a_g1"], hd["b_g1"], hd["b_g2"], hd["l_g1"], hd["h_g1"]], [n, n, n, n, n - 1], [0] * 5)
        cuts = [0, n // 3, n // 2, n]
        for r in range(3):
            lo, hi = cuts[r], cuts[r + 1]
            wm, hm = w.clone(), h.clone()
            wm[:4 * lo] = 0; wm[4 * hi:] = 0
            hm[:4 * lo] = 0; hm[4 * hi:] = 0
            ctx.groth16_commit_partial(pk, wm, hm, None, None, blocks[96 * r:], F.G16_INPUTS_DEVICE | F.G16_H_COEFFS)
        assert ctx.groth16_fold(blocks, 3) == (whole, b1_whole)
    finally:
        circuit.close()


def test_groth16_with_columns_left_on_plain_bases(ctx, monkeypatch):
    """A key too large for window tables on every column (domain 2^24 on an 80 GB GPU) keeps some columns on plain
    bases: the one-call prove over mixed plans and the separate calls still give the proof of an all-plain key."""
    import torch
    from ethrex_b200.groth16 import SyntheticWrapCircuit
    log_n = 10
    plain = SyntheticWrapCircuit(ctx, log_n, precompute=False)
    try:
        ref = plain.prove_device(b"batch-1")
    finally:
        plain.close()
    # a workspace reserve no device can meet: only the first column gets its table
    monkeypatch.setattr(SyntheticWrapCircuit, "PROVE_WORKSPACE_PER_POINT", torch.cuda.mem_get_info()[1] // (1 << log_n) + 1)
    circuit = SyntheticWrapCircuit(ctx, log_n, precompute=True)
    try:
        assert circuit.plain_columns == ["b_g1", "b_g2", "l_g1", "h_g1"]
        assert circuit.prove_device(b"batch-1") == ref
        assert circuit.prove_separate(b"batch-1")[0] == ref[0]
    finally:
        circuit.close()


def test_groth16_commit_rejects_inconsistent_keys(ctx):
    from ethrex_b200.groth16 import SyntheticWrapCircuit
    circuit = SyntheticWrapCircuit(ctx, 6, precompute=False)
    try:
        hd = circuit.pk.handles
        n = 64
        w, a, b, c = circuit.assign(b"x")
        good = [hd["a_g1"], hd["b_g1"], hd["b_g2"], hd["l_g1"], hd["h_g1"]]
        from ethrex_b200 import _ffi as F
        for handles, counts, offsets in (
            ([hd["b_g2"]] + good[1:], [n] * 4 + [n - 1], [0] * 5),   # a G2 handle in a G1 column
            (good, [n + 1, n, n, n, n - 1], [0] * 5),                 # more scalars than resident points
            (good, [n] * 4 + [n], [0, 0, 0, 0, 1]),                   # H reaches past the quotient's coefficients
            ([0] + good[1:], [n] * 4 + [n - 1], [0] * 5),             # only B_g1 may be absent
        ):
            with pytest.raises(eb.B200Error):
                ctx.groth16_commit(ctx.groth16_pk(6, handles, counts, offsets), w, a, b, c, F.G16_INPUTS_DEVICE)
        # B_g1 absent: same proof, [B]1 reported as the identity
        w, a, b, c = circuit.assign(b"x")
        ref, _ = circuit.prove_device(b"x")
        proof, b1 = ctx.groth16_commit(ctx.groth16_pk(6, [good[0], 0] + good[2:], [n] * 4 + [n - 1], [0] * 5), w, a, b, c, F.G16_INPUTS_DEVICE)
        assert proof == ref and b1 == bytes(64)
    finally:
        circuit.close()


def test_verifier_rejects_non_canonical_encodings(ctx):
    """ADVICE r1 (medium): A = (x, y + p) and a public input x + r must NOT verify (the levm ecpairing wrapper and the
    on-chain verifier reject the first, /root/reference/crates/vm/levm/src/precompiles.rs:801-820; the second is
    public-input aliasing)."""
    from ethrex_b200.groth16 import Groth16Prover, Groth16Verifier
    from groth16_toy import N_PUBLIC, ToyGroth16, _g1
    toy = ToyGroth16(3)
    prover = Groth16Prover(ctx, 3, toy.a_g1, toy.b_g1, toy.b_g2, toy.l_g1, toy.h_g1, N_PUBLIC)
    ver = Groth16Verifier(ctx, toy.vk_alpha_g1, toy.vk_beta_g2, toy.vk_gamma_g2, toy.vk_delta_g2, [_g1(s) for s in toy.ic])
    try:
        x = 77
        z = toy.assign(x)
        proof = prover.prove(z, *toy.evaluations(z))
        assert proof == toy.expected_proof(z)
        assert ver.verify(proof, [x])
        ay = int.from_bytes(proof[32:64], "big")
        assert ay + pyref.P < (1 << 256)
        forged = proof[:32] + (ay + pyref.P).to_bytes(32, "big") + proof[64:]
        assert not ver.verify(forged, [x])
        assert not ver.verify(proof, [x + pyref.R])
        assert not ver.verify(proof, [-1])
        assert ver.verify_batch([proof, forged, proof], [[x], [x], [x + pyref.R]]) == [True, False, False]
    finally:
        prover.close()


@pytest.mark.parametrize("table", [False, True])
def test_two_level_sort_on_skewed_scalars(ctx, table):
    """The r2 sort (n >= 2^16) under the distributions that break naive bucket sorts (SURVEY.md section 8d): all scalars equal
    (13 buckets hold everything: one coarse bin per window), half zeros, tiny scalars (only window 0 populated), r - 1, and a
    Zipf-like mix -- each against the CPU oracle's Pippenger.  The fine pass works on fixed segments of a bin, so a heavy
    bin costs time, not correctness or one CTA's patience."""
    n = (1 << 17) + 12345
    k, d = chain_kd()
    pts = orc.g1_chain(n, k, d)
    dp = to_dev(pts)
    rnd = orc.rand_fr(pyref.SEED_SCALARS, 0, n)
    cases = {}
    eq = np.tile(rnd[5], (n, 1)); cases["all equal"] = eq
    hz = rnd.copy(); hz[::2] = 0; cases["half zeros"] = hz
    tiny = np.zeros((n, 4), dtype=np.uint64); tiny[:, 0] = rnd[:, 0] & np.uint64(0xFFFF); cases["below 2^16"] = tiny
    rm1 = np.tile(orc.int_to_limbs(pyref.R - 1), (n, 1)); cases["all r - 1"] = rm1
    zipf = rnd.copy(); zipf[: n // 2] = rnd[7]; zipf[n // 2: 3 * n // 4] = rnd[11]; cases["zipf-like"] = zipf
    h = None
    try:
        if table:
            h = ctx.g1_bases_from_device(dp, n)
            ctx.bases_precompute(h, 0)
        for name, s in cases.items():
            s = np.ascontiguousarray(s)
            exp = orc.g1_msm(pts, s)
            got = ctx.g1_msm_resident_device(h, to_dev(s), n) if table else ctx.g1_msm_device(dp, to_dev(s), n)
            assert got == exp, name
    finally:
        if h is not None:
            ctx.bases_free(h)


def test_host_scalar_pipeline_with_growing_chunks(ctx, monkeypatch):
    """b200zk_g1_msm_resident with HOST scalars cuts the points into chunks whose sizes grow geometrically (only the first
    chunk's upload is exposed; B200ZK_CHUNK_RATIO, default 3; set_msm_chunks = how many).  Every (count, ratio) -- equal
    chunks, steep growth, more chunks than 1024-point units at the small size -- must return the one-shot bytes, with the
    two-level sort (chunks >= 2^16 points) and with the legacy one (small chunks), on plain bases and on a window table."""
    k, d = chain_kd()
    n = (1 << 18) + 777
    pts = orc.g1_chain(n, k, d)
    s = np.ascontiguousarray(orc.rand_fr(pyref.SEED_SCALARS, 0, n))
    s[: n // 3] = s[3]                       # a heavy bucket per window inside the first chunks
    exp = orc.g1_msm(pts, s)
    dp = to_dev(pts)
    h = ctx.g1_bases_from_device(dp, n)
    ht = ctx.g1_bases_from_device(dp, n)
    ctx.bases_precompute(ht, 0)
    try:
        assert ctx.g1_msm_resident_device(ht, to_dev(s), n) == exp
        for chunks in (2, 3, 5):
            ctx.set_msm_chunks(chunks)
            for ratio in ("1", "2.5", "3", "8"):
                monkeypatch.setenv("B200ZK_CHUNK_RATIO", ratio)
                assert ctx.g1_msm_resident(ht, s, n) == exp, (chunks, ratio, "table")
                assert ctx.g1_msm_resident(h, s, n) == exp, (chunks, ratio, "plain")
                m = 5000                      # tiny: most chunks are empty and vanish
                assert ctx.g1_msm_resident(h, s[:m], m) == orc.g1_msm(pts[:m], s[:m]), (chunks, ratio, "tiny")
    finally:
        ctx.set_msm_chunks(0)
        ctx.bases_free(h)
        ctx.bases_free(ht)
