"""Groth16 from circom artifacts on the device (b200zk_groth16_zkey_*, ethrex_b200.zkey.ZkeyProver): snarkjs-layout files
of tests/zkey_ref.py proved bit-exactly against the proof in the exponent, verified under the key's own verifying key,
and tied to the shipped prover (b200zk_groth16_prove over the same QAP in the ark layout, fed host evaluations) at
larger domains, one of them with a row of 10^5 terms; then every device-side refusal, each followed by a good proof."""
import random
import struct

import numpy as np
import pytest

import cpu_oracle as orc
import pyref as o
import zkey_ref as zr

import ethrex_b200 as eb
from ethrex_b200 import _ffi as F
from ethrex_b200.groth16 import Groth16ZkProver
from ethrex_b200.zkey import ZkeyProver

pytestmark = pytest.mark.gpu

R = zr.R
RS = {"zero": (0, 0), "random": (0x2B1E4D7F9A3C6E8B0D2F4A6C8E0B3D5F7A9C1E3B5D7F9A2C4E6B8D0F2A4C6E8, 0x1D3F5B7E9A2C4E6B8D0F2A4C6E8B1D3F5A7C9E0B2D4F6A8C0E2B4D6F8A1C3E5),
      "order_minus_1": (R - 1, R - 1)}
_CIRCUITS = {}


def _circuit(n_constraints, n_public):
    key = (n_constraints, n_public)
    if key not in _CIRCUITS:
        c = zr.ZkeyCircuit(n_constraints, n_public, seed=0x5EED + n_constraints)
        _CIRCUITS[key] = (c, c.zkey())
    return _CIRCUITS[key]


def _public(n_public):
    return [0x1234567 + 11 * i for i in range(n_public)]


@pytest.mark.parametrize("case", sorted(RS))
@pytest.mark.parametrize("shape", [(5, 1), (11, 2), (27, 3)])
@pytest.mark.parametrize("precompute", [False, True])
def test_proof_equals_the_exponent(ctx, shape, case, precompute):
    c, zkey = _circuit(*shape)
    r, s = RS[case]
    prover = ZkeyProver(ctx, zkey, precompute=precompute)
    try:
        assert (prover.n_vars, prover.n_public, prover.log_n) == (c.n_vars, c.n_public, c.log_n)
        z = c.assign(_public(c.n_public))
        assert prover.prove(c.wtns(z), r=r, s=s) == c.expected_proof(z, r, s)
    finally:
        prover.close()


def test_proofs_verify_under_the_keys_vk(ctx):
    c, zkey = _circuit(11, 2)
    prover = ZkeyProver(ctx, zkey)
    try:
        assert prover.vk == c.vk()
        ver = prover.verifier()
        pub = _public(2)
        w = c.wtns(c.assign(pub))
        proofs = [prover.prove(w, r=r, s=s) for r, s in RS.values()] + [prover.prove(w), prover.prove(w)]
        assert len(set(proofs)) == len(proofs)
        assert all(ver.verify_batch(proofs, [pub] * len(proofs)))
        assert not any(ver.verify_batch(proofs, [[pub[0] + 1, pub[1]]] * len(proofs)))
        # a different witness of the same circuit
        pub2 = [5, 6]
        assert ver.verify(prover.prove(c.wtns(c.assign(pub2))), pub2)
    finally:
        prover.close()


# ---- agreement with b200zk_groth16_prove over the same QAP ----------------------------------------------------------------
def _g1_mul_batch(ctx, scalars):
    """[k]G for each k, EIP-196 bytes, on the device"""
    g = o.g1_to_be(o.G1_GEN)
    out, st = ctx.bn254_g1_mul_batch(g * len(scalars), b"".join((k % R).to_bytes(32, "big") for k in scalars))
    assert all(x in (0, 1) for x in st)
    return out


def _batch_inv(vals):
    pre, acc = [], 1
    for v in vals:
        pre.append(acc)
        acc = acc * v % R
    inv = pow(acc, -1, R)
    out = [0] * len(vals)
    for i in range(len(vals) - 1, -1, -1):
        out[i] = inv * pre[i] % R
        inv = inv * vals[i] % R
    return out


class BigPair:
    """a random sparse QAP at domain 2^log_n as a .zkey and as the ark-layout key of Groth16ZkProver, sharing tau and delta
    and the column points (chains); the witness need not satisfy the rows (c = a o b on the domain, so a b - c vanishes
    there whatever a and b are).  long_row: terms of one extra A row, next to the 2^(log_n - 1) short rows."""

    def __init__(self, ctx, log_n, n_vars, long_row=0, seed=7):
        import torch
        rng = random.Random(seed)
        n = 1 << log_n
        self.log_n, self.n, self.n_vars, self.n_public = log_n, n, n_vars, 2
        recs = []
        for j in range(n // 2):
            for m in (0, 1):
                for _ in range(rng.randrange(1, 4)):
                    recs.append((m, j, rng.randrange(n_vars), rng.randrange(R)))
        for _ in range(long_row):
            recs.append((0, n // 2, rng.randrange(n_vars), rng.randrange(R)))
        for i in range(self.n_public + 1):
            recs.append((0, n // 2 + 1 + i, i, 1))
        rng.shuffle(recs)
        self.z = [1] + [rng.randrange(R) for _ in range(n_vars - 1)]
        a, b = [0] * n, [0] * n
        for m, j, i, cf in recs:
            if m == 0: a[j] = (a[j] + cf * self.z[i]) % R
            else: b[j] = (b[j] + cf * self.z[i]) % R
        self.evals = (a, b, [x * y % R for x, y in zip(a, b)])
        # column points: chains computed on the device, native bytes for the zkey and BE bytes for the ark key
        cols = {}
        for name, g2, cnt, kk in (("a", False, n_vars, 3), ("b1", False, n_vars, 5), ("b2", True, n_vars, 7), ("c", False, n_vars - 3, 11)):
            pts = torch.empty((16 if g2 else 8) * cnt, dtype=torch.int64, device="cuda")
            (ctx.g2_chain_device if g2 else ctx.g1_chain_device)(pts, 0, cnt, kk, 2 * kk + 1)
            nat = pts.cpu().numpy().view(np.uint64).reshape(cnt, 16 if g2 else 8)
            cols[name] = (nat.tobytes(), (orc.g2_native_to_be if g2 else orc.g1_native_to_be)(nat))
        tau, delta = rng.randrange(2, R), rng.randrange(2, R)
        alpha, beta, gamma = rng.randrange(2, R), rng.randrange(2, R), rng.randrange(2, R)
        dinv = pow(delta, -1, R)
        # zkey H: L_{2i+1}(tau) / delta over the doubled domain; ark H: tau^i Z(tau) / delta, i < n - 1
        w2 = o.root_of_unity(log_n + 1)
        z2 = (pow(tau, 2 * n, R) - 1) * pow(2 * n, -1, R) % R
        wk, step, ks = w2, w2 * w2 % R, []
        for _ in range(n):
            ks.append(wk)
            wk = wk * step % R
        invs = _batch_inv([(tau - k) % R for k in ks])
        h_zkey = _g1_mul_batch(ctx, [z2 * k % R * iv % R * dinv % R for k, iv in zip(ks, invs)])
        zt = (pow(tau, n, R) - 1) % R
        hs, t = [], zt * dinv % R
        for _ in range(n - 1):
            hs.append(t)
            t = t * tau % R
        h_ark = _g1_mul_batch(ctx, hs)
        terms = {"alpha1": zr._g1(alpha), "beta1": zr._g1(beta), "beta2": zr._g2(beta), "gamma2": zr._g2(gamma), "delta1": zr._g1(delta), "delta2": zr._g2(delta)}
        g1n = lambda be: orc.g1_be_to_native(be).tobytes()  # noqa: E731
        g2n = lambda be: orc.g2_be_to_native(be).tobytes()  # noqa: E731
        hdr = struct.pack("<I", 32) + zr.P.to_bytes(32, "little") + struct.pack("<I", 32) + R.to_bytes(32, "little") + struct.pack("<III", n_vars, 2, n)
        hdr += g1n(terms["alpha1"]) + g1n(terms["beta1"]) + g2n(terms["beta2"]) + g2n(terms["gamma2"]) + g1n(terms["delta1"]) + g2n(terms["delta2"])
        ic = b"".join(zr.g1_native(k) for k in (1, 2, 3))
        self.zkey = zr.container(b"zkey", 1, [(1, struct.pack("<I", 1)), (2, hdr), (3, ic),
                                             (4, struct.pack("<I", len(recs)) + b"".join(zr.coef_record(*r) for r in recs)),
                                             (5, cols["a"][0]), (6, cols["b1"][0]), (7, cols["b2"][0]), (8, cols["c"][0]), (9, g1n(h_zkey))])
        self.wtns = zr.wtns_bytes(self.z)
        self.ark = (cols["a"][1], cols["b1"][1], cols["b2"][1], cols["c"][1], h_ark)
        self.terms = (terms["alpha1"], terms["beta1"], terms["beta2"], terms["delta1"], terms["delta2"])


def _agree(ctx, pair):
    zp = ZkeyProver(ctx, pair.zkey)
    ark = Groth16ZkProver(ctx, pair.log_n, *pair.ark, pair.n_public + 1, *pair.terms)
    try:
        for r, s in RS.values():
            assert zp.prove(pair.wtns, r=r, s=s) == ark.prove(pair.z, *pair.evals, r=r, s=s)
    finally:
        zp.close()
        ark.close()


def test_agrees_with_the_existing_prover_small(ctx):
    """the oracle's circuit in both layouts (its own H columns), same r, s"""
    c, zkey = _circuit(27, 3)
    z = c.assign(_public(3))
    zp = ZkeyProver(ctx, zkey)
    dinv = pow(c.delta, -1, R)
    zt = (pow(c.tau, c.n, R) - 1) % R
    cols = (b"".join(zr._g1(x) for x in c.u), b"".join(zr._g1(x) for x in c.v), b"".join(zr._g2(x) for x in c.v),
            b"".join(zr._g1(c.k[i] * dinv) for i in range(c.n_public + 1, c.n_vars)),
            b"".join(zr._g1(pow(c.tau, i, R) * zt * dinv) for i in range(c.n - 1)))
    terms = (zr._g1(c.alpha), zr._g1(c.beta), zr._g2(c.beta), zr._g1(c.delta), zr._g2(c.delta))
    ark = Groth16ZkProver(ctx, c.log_n, *cols, c.n_public + 1, *terms)
    try:
        for r, s in RS.values():
            assert zp.prove(c.wtns(z), r=r, s=s) == ark.prove(z, *c.evaluations(z), r=r, s=s) == c.expected_proof(z, r, s)
    finally:
        zp.close()
        ark.close()


def test_skewed_rows_agree_with_the_existing_prover(ctx):
    """2^16 short rows and one row of 10^5 terms (domain 2^17)"""
    _agree(ctx, BigPair(ctx, 17, 4096, long_row=100_000))


def test_domain_2_20_agrees_with_the_existing_prover(ctx):
    _agree(ctx, BigPair(ctx, 20, 1 << 16, seed=20))


# ---- refusals on the device -------------------------------------------------------------------------------------------------
def _load_status(ctx, data):
    import ctypes as C
    h = C.c_uint64()
    buf = C.create_string_buffer(bytes(data), len(data))
    rc = F.lib.b200zk_groth16_zkey_load(ctx._h, buf, len(data), 0, C.byref(h))
    if rc == F.OK:
        F.lib.b200zk_groth16_zkey_free(ctx._h, h.value)
    return rc, F.lib.b200zk_last_error(ctx._h).decode()


def test_refusals_leave_the_context_usable(ctx):
    c, zkey = _circuit(11, 2)
    secs = c.sections()
    z = c.assign(_public(2))
    good = c.expected_proof(z, 3, 4)
    prover = ZkeyProver(ctx, zkey)

    def still_good():
        assert prover.prove(c.wtns(z), r=3, s=4) == good

    def patched(sid, off, blob):
        return zr.container(b"zkey", 1, [(i, p[:off] + blob + p[off + len(blob):] if i == sid else p) for i, p in secs])

    try:
        one_mont = ((1 << 256) % zr.P).to_bytes(32, "little")
        cases = [
            (patched(5, 64 * 4, one_mont + one_mont), F.ERR_NOT_ON_CURVE, "section 5 (A): point 4 is not on the curve"),
            (patched(7, 128 * 2 + 32, one_mont), F.ERR_NOT_ON_CURVE, "section 7 (B2): point 2"),
            (patched(2, 84, one_mont + one_mont), F.ERR_NOT_ON_CURVE, "alpha1 is not on the curve"),
            (patched(3, 64, one_mont + one_mont), F.ERR_NOT_ON_CURVE, "section 3 (IC): point 1"),
            (patched(9, 64 * 3 + 32, zr.P.to_bytes(32, "little")), F.ERR_NOT_IN_FIELD, "section 9 (H): point 3 has a coordinate >= q"),
            (patched(8, 0, ((1 << 256) - 1).to_bytes(32, "little")), F.ERR_NOT_IN_FIELD, "section 8 (C): point 0"),
            (zr.container(b"zkey", 1, c.sections(c.records()[:4] + [(0, c.n, 1, 5)])), F.ERR_INVALID_ARG, "record 4: constraint >= domainSize"),
            (zr.container(b"zkey", 1, c.sections(c.records()[:2] + [(1, 0, c.n_vars, 5)])), F.ERR_INVALID_ARG, "record 2: signal >= nVars"),
            (zr.container(b"zkey", 1, c.sections([(2, 0, 1, 5)])), F.ERR_INVALID_ARG, "record 0: matrix"),
            (zkey[:-1], F.ERR_INVALID_ARG, "truncated"),
        ]
        for data, st, frag in cases:
            rc, msg = _load_status(ctx, data)
            assert rc == st and frag in msg, (rc, msg)
            still_good()
        # witness value >= r; r or s >= r
        bad = list(z)
        bad[5] = R
        with pytest.raises(eb.B200Error, match="value 5 is >= r"):
            prover.prove(zr.wtns_bytes(bad), r=3, s=4)
        still_good()
        for r, s in ((R, 0), (0, R), (1 << 255, 1)):
            with pytest.raises(eb.B200Error, match="r or s"):
                prover.prove(c.wtns(z), r=r, s=s)
            still_good()
        with pytest.raises(eb.B200Error, match="nWitness"):
            prover.prove(zr.wtns_bytes(z[:-1]), r=3, s=4)
        still_good()
        # the halo2 root: the odd coset would be another one
        ctx.set_ntt_root(ctx.ntt_root_preset(ctx.NTT_ROOT_HALO2))
        try:
            with pytest.raises(eb.B200Error, match="NTT root is not preset 0"):
                prover.prove(c.wtns(z), r=3, s=4)
        finally:
            ctx.set_ntt_root(None)
        still_good()
        assert F.lib.b200zk_groth16_zkey_free(ctx._h, prover.key + 1000) == F.ERR_INVALID_ARG
    finally:
        prover.close()


def test_proof_verifies_under_the_python_pairing(ctx):
    """the device proof against the key's vk through the oracle's pairing, independent of the device pairing"""
    c, zkey = _circuit(11, 2)
    prover = ZkeyProver(ctx, zkey)
    try:
        pub = _public(2)
        proof = prover.prove(c.wtns(c.assign(pub)), r=RS["random"][0], s=RS["random"][1])
        vk = prover.vk
        ic = [o.g1_from_be(vk[448 + 64 * i: 512 + 64 * i]) for i in range(3)]
        vk_x = ic[0]
        for x, p in zip(pub, ic[1:]):
            vk_x = o.g1_add(vk_x, o.g1_mul(x, p))
        a, b, cc = o.g1_from_be(proof[:64]), o.g2_from_be(proof[64:192]), o.g1_from_be(proof[192:])
        alpha, beta, gamma, delta = o.g1_from_be(vk[:64]), o.g2_from_be(vk[64:192]), o.g2_from_be(vk[192:320]), o.g2_from_be(vk[320:448])
        neg_a = o.pt_neg(o._Fq, a)
        assert o.pairing_check([(neg_a, b), (alpha, beta), (vk_x, gamma), (cc, delta)])
        wrong = o.g1_add(vk_x, ic[1])  # the first public input plus one
        assert not o.pairing_check([(neg_a, b), (alpha, beta), (wrong, gamma), (cc, delta)])
    finally:
        prover.close()


def test_key_loaded_under_another_ntt_root_proves_under_preset_0(ctx):
    """the odd coset's generator comes from the preset-0 root, not from the root the context holds at load time"""
    c, zkey = _circuit(11, 2)
    z = c.assign(_public(2))
    ctx.set_ntt_root(ctx.ntt_root_preset(ctx.NTT_ROOT_HALO2))
    try:
        prover = ZkeyProver(ctx, zkey)
    finally:
        ctx.set_ntt_root(None)
    try:
        assert prover.prove(c.wtns(z), r=3, s=4) == c.expected_proof(z, 3, 4)
    finally:
        prover.close()


def test_load_and_free_return_device_memory(ctx):
    import torch
    pair = BigPair(ctx, 16, 1 << 14, seed=16)
    for _ in range(2):  # the context's workspaces grow once
        p = ZkeyProver(ctx, pair.zkey)
        p.prove(pair.wtns, r=1, s=2)
        p.close()
    ctx.synchronize()
    before = torch.cuda.mem_get_info()[0]
    for _ in range(4):
        p = ZkeyProver(ctx, pair.zkey)
        p.prove(pair.wtns, r=1, s=2)
        p.close()
    ctx.synchronize()
    assert abs(torch.cuda.mem_get_info()[0] - before) < 8 << 20
