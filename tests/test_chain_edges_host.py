"""The chain tracers and edge constructors of tests/chain_edges_ref.py on the CPU: each tracer computes what the oracles
compute, each constructed input meets its event at its step, the raw-scalar enumeration is complete, and the constructed
inputs agree with independent anchors (OpenSSL through `cryptography`, the affine pairing of bls_pairing_ref)."""
import random

import pytest
from cryptography.exceptions import InvalidSignature
from cryptography.hazmat.primitives import hashes
from cryptography.hazmat.primitives.asymmetric import ec, utils

import bls12_map_ref as M
import bls12_ops_ref as ops
import bls_pairing_ref as B
import bls_ref as bls
import chain_edges_ref as E
import pyref
import secp256k1_ref as k1
import secp256r1_ref as r1

CURVES = {"bn254_g1": (pyref.R, E.BN_G1, pyref.G1_GEN, pyref.g1_mul), "bls12_381_g1": (bls.R, E.BLS_G1, bls.G1, ops.G1.mul),
          "bls12_381_g2": (bls.R, E.BLS_G2, B.G2, ops.G2.mul)}


@pytest.fixture(scope="module")
def maps():
    return E.map_cases()


# ---- raw-scalar chains ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("curve, cells", [("bn254_g1", {(1, 0), (1, 1), (1, 2), (3, 0), (5, 0)}), ("bls12_381_g1", {(1, 0), (1, 1)})])
def test_raw_scalar_enumeration_is_complete(curve, cells):
    r = CURVES[curve][0]
    edges = E.raw_scalar_edges(r, 7)
    assert {ms for _, _, _, ms in edges} == cells
    # brute force over every prefix near a multiple of r below 2^256: the add at odd prefix A meets (A - 1) P + P
    prefixes = E.exceptional_prefixes(r)
    for q in range((1 << 256) // r + 1):
        for a in range(max(1, q * r - 6), q * r + 7):
            if a & 1 and a < 1 << 256:
                assert (E.kind(E.Logs(r), (a - 1) % r, 1) in (E.DOUBLE, E.CANCEL)) == (a in prefixes)
    # every (A, s) with A 2^s < 2^256 is enumerated, and random scalars meet events only at those prefixes
    want = {(a, s) for a in prefixes for s in range(256) if a << s < 1 << 256}
    assert {(k >> s, s) for k, _, s, _ in edges} == want
    rng = random.Random(1)
    for k in [rng.randrange(1 << 256) for _ in range(3000)] + [rng.randrange(r, 1 << 256) | 1 for _ in range(3000)]:
        _, tr = E.run(E.scalar_mul, E.Logs(r), k, 1)
        assert all((k >> i, i) in want for (_, i), _ in tr.exceptional())


@pytest.mark.parametrize("curve", ["bn254_g1", "bls12_381_g1"])
def test_raw_scalar_edges_meet_their_event(curve):
    r = CURVES[curve][0]
    reseeded = 0
    for k, kd, step, label in E.scalar_cases(curve):
        _, tr = E.run(E.scalar_mul, E.Logs(r), k, 1)
        if step is None:
            assert tr.exceptional() == [], label
            continue
        assert tr.exceptional() == [(step, kd)], label
        after = [ev for ev in tr.events if ev[0][1] < step[1]]
        if kd == E.CANCEL and k & ((1 << step[1]) - 1):  # identity, then the next set bit reseeds the accumulator
            assert after[0][1] == E.IDENTITY, label
            reseeded += 1
    assert reseeded >= 1


def test_endomorphism_eigenvalues():
    lams = E.endomorphism_eigenvalues()
    for name in ("bn254_g1", "bls12_381_g1"):
        r = CURVES[name][0]
        assert len(lams[name]) == 2 and all((lam * lam + lam + 1) % r == 0 for lam in lams[name])
    assert lams["bls12_381_g2"] == [-M.Z_ABS % bls.R]  # p = z (mod r) for BLS12 curves


@pytest.mark.parametrize("curve", list(CURVES))
def test_scalar_mul_tracer_equals_the_oracle(curve):
    """the tracer over real points equals the oracle's k P and records what the discrete-log tracer records"""
    r, g, gen, mul = CURVES[curve]
    rng = random.Random(2)
    p = mul(rng.randrange(1, r), gen)
    ks = [k for k, *_ in E.scalar_cases("bls12_381_g1" if curve == "bls12_381_g2" else curve)] + [rng.randrange(1 << 256) for _ in range(4)]
    if curve == "bls12_381_g2":
        ks = ks[:6] + E.endomorphism_eigenvalues()[curve] + ks[-2:]
    for k in ks:
        v, tr = E.run(E.scalar_mul, g, k, p)
        _, tl = E.run(E.scalar_mul, E.Logs(r), k, 1)
        assert v == mul(k % r, p) and tr.events == tl.events, hex(k)


# ---- the ECDSA ladder ---------------------------------------------------------------------------------------------------------
def _ladder_check(case, n, g, gen, derive, oracle_point):
    p = case.params
    _, tl = E.run(E.lincomb, E.Logs(n), p["u1"], p["u2"], p["t"], 1)
    assert ((p["op"], p["i"]), p["kind"]) in tl.events and [ev for ev in tl.exceptional() if ev[0] != (p["op"], p["i"])] == [], case.label
    u1, u2, R = derive(case.data)
    assert (u1, u2) == (p["u1"], p["u2"]) and R == g.mul(p["t"], gen)
    v, tr = E.run(E.lincomb, g, u1, u2, R, gen)
    assert tr.events == tl.events and v == g.mul((u1 + u2 * p["t"]) % n, gen) and v == oracle_point(case.data), case.label
    return tl


def test_ecrecover_ladder_cases():
    through_o = 0
    for c in E.ecrecover_cases():
        tl = _ladder_check(c, k1.N, E.K1, k1.G, lambda d: E.ecrecover_ladder(d[:65], d[65:]), lambda d: k1.recover_point(d[:65], d[65:])[1])
        at = tl.events.index((c.step, c.event))
        through_o += c.event == E.CANCEL and any(k == E.IDENTITY for _, k in tl.events[at + 1:])  # O, then reseeded
    assert {(c.step[0], c.event) for c in E.ecrecover_cases()} == {(op, kd) for op in "RG" for kd in (E.DOUBLE, E.CANCEL)}
    assert through_o >= 3


def test_p256_ladder_cases():
    for c in E.p256_cases():
        def oracle(d):
            u1, u2, q = E.p256_ladder(d)
            return r1.lincomb(u1, r1.G, u2, q)
        _ladder_check(c, r1.N, E.R1, r1.G, E.p256_ladder, oracle)


def test_ladder_tracer_on_random_inputs():
    rng = random.Random(3)
    for _ in range(8):
        u1, u2, t = rng.randrange(1, k1.N), rng.randrange(1, k1.N), rng.randrange(1, k1.N)
        v, tr = E.run(E.lincomb, E.K1, u1, u2, k1.mul(t, k1.G), k1.G)
        assert v == k1.add(k1.mul(u1, k1.G), k1.mul(u2 * t % k1.N, k1.G)) and tr.exceptional() == []
        v, _ = E.run(E.lincomb, E.R1, u1 % r1.N, u2 % r1.N, r1.mul(t, r1.G), r1.G)
        assert v == r1.lincomb(u1 % r1.N, r1.G, u2 % r1.N, r1.mul(t, r1.G))


def test_p256_cases_against_openssl():
    """OpenSSL accepts exactly the constructed signatures the oracle accepts"""
    verdicts = []
    for c in E.p256_cases():
        h, r, s, qx, qy = r1.decode(c.data)
        key = ec.EllipticCurvePublicNumbers(qx, qy, ec.SECP256R1()).public_key()
        try:
            key.verify(utils.encode_dss_signature(r, s), h.to_bytes(32, "big"), ec.ECDSA(utils.Prehashed(hashes.SHA256())))
            ok = True
        except InvalidSignature:
            ok = False
        assert ok == r1.verify(c.data), c.label
        verdicts.append(ok)
    assert True in verdicts and False in verdicts


def test_ecrecover_cases_against_openssl():
    """every recovery with status 0 verifies under the recovered key"""
    statuses = []
    for c in E.ecrecover_cases():
        sig, msg = c.data[:65], c.data[65:]
        st, q = k1.recover_point(sig, msg)
        statuses.append(st)
        if st == 0:
            key = ec.EllipticCurvePublicNumbers(q[0], q[1], ec.SECP256K1()).public_key()
            key.verify(utils.encode_dss_signature(int.from_bytes(sig[:32], "big"), int.from_bytes(sig[32:64], "big")), msg,
                       ec.ECDSA(utils.Prehashed(hashes.SHA256())))
    assert set(statuses) == {0, 3}


# ---- map-to-curve -------------------------------------------------------------------------------------------------------------
def test_isogenous_curves_have_the_group_orders():
    rng = random.Random(4)
    for curve in (E.E1, E.E2):
        for _ in range(3):
            p = curve.random_point(rng)
            assert curve.on_curve(p) and curve.mul(curve.order, p) is None
            assert all(curve.mul(curve.order // ell, p) is not None for ell in (bls.R,))
        assert curve.on_curve(curve.add(p, curve.add(p, p)))


def test_inverse_sswu():
    rng = random.Random(5)
    for curve, u in ((E.E1, rng.randrange(M.P)), (E.E2, (rng.randrange(M.P), rng.randrange(M.P)))):
        x, _ = curve.sswu(u)
        us = curve.preimages(x)
        assert u in us and all(curve.sswu(v)[0] == x for v in us)


def test_g1_isogeny_kernel_preimages():
    """x_den of the 11-isogeny has 5 roots in Fp; the 2 with a point on E' have 8 SSWU preimages each"""
    inputs = E.g1_kernel_inputs()
    assert len(inputs) == 5 and sorted(len(us) for us in inputs.values()) == [0, 0, 0, 8, 8]
    for x0, us in inputs.items():
        for u in us:
            x, y = E.E1.sswu(u)
            assert x == x0 and M.iso_map(M.Fp, M.G1_TABLES, (x, y)) is None
            assert M.map_fp_to_g1_bytes(M.fp64(u)) == (bytes(128), 1)


def test_g2_isogeny_kernel_is_unreachable():
    """x_den of the 3-isogeny has one double root x0 in Fp2 and x0^3 + A' x0 + B' is not a square: no point of E2' has x0"""
    _, g = E.g2_kernel_root()
    assert M.Fp2.sqrt(g) is None


def test_torsion_inputs(maps):
    """every prime of both cofactors but 3 (whose only x on E' has no preimage) gives inputs, at every l-power order met"""
    g1, g2, (c1, c2) = maps
    assert {ell for (ell, _), n in c1.items() if n} == set(E.E1.primes) - {3} and c1[(3, 1)] == 0
    assert {ell for (ell, _), n in c2.items() if n} == set(E.E2.primes)
    assert c1[(11, 2)] > 0  # E'(Fp) holds points of order 121
    assert len(g1) == 16 + sum(c1.values()) and len(g2) == sum(c2.values())


@pytest.mark.parametrize("group", ["g1", "g2"])
def test_map_cases_reach_infinity(maps, group):
    """each constructed u maps to the identity in the oracle and in the tracer of the device's chain; a doubling inside
    mul_u64 is among them"""
    cases = maps[0] if group == "g1" else maps[1]
    tracer, g, oracle, size = (E.map_g1, E.BLS_G1, M.map_fp_to_g1_bytes, 128) if group == "g1" else (E.map_g2, E.BLS_G2, M.map_fp2_to_g2_bytes, 256)
    kinds = set()
    for c in cases:
        if c.params["ell"] is not None:
            curve = E.E1 if group == "g1" else E.E2
            pt = curve.sswu(c.params["u"])
            assert curve.mul(c.params["ell"] ** c.params["k"], pt) is None and curve.mul(c.params["ell"] ** (c.params["k"] - 1), pt) is not None
        v, tr = E.run(tracer, g, c.params["u"])
        assert v is None and oracle(c.data) == (bytes(size), 1), c.label
        kinds |= {(s[0], k) for s, k in tr.exceptional()}
    if group == "g1":
        assert ("heff", E.DOUBLE) in kinds and ("heff", E.CANCEL) in kinds
    else:
        assert ("psi", E.CANCEL) in kinds and ("z1", E.CANCEL) in kinds


def test_map_tracers_equal_the_oracle_on_random_u():
    rng = random.Random(6)
    for _ in range(6):
        u = rng.randrange(M.P)
        assert E.run(E.map_g1, E.BLS_G1, u)[0] == M.map_to_g1(u)
    for _ in range(3):
        u = (rng.randrange(M.P), rng.randrange(M.P))
        v, tr = E.run(E.map_g2, E.BLS_G2, u)
        assert v == M.map_to_g2(u) == M.clear_cofactor_g2_scalar(M.iso_map(M.Fp2, M.G2_TABLES, M.sswu(M.Fp2, M.G2_A, M.G2_B, M.G2_Z, u)))
        assert tr.exceptional() == []


# ---- point evaluation ---------------------------------------------------------------------------------------------------------
def _combine(p):
    return E.run(E.kzg_combine, E.Logs(bls.R), p["c"], p["z"], p["y"], p["a"], 1)


def test_kzg_cases_meet_their_event():
    cases = E.kzg_cases()
    assert {(c.step, c.event) for c in cases} == {(s, k) for s in (("C", 0), ("-yG", 0)) for k in (E.DOUBLE, E.CANCEL)}
    for c in cases:
        p = c.params
        v, tr = _combine(p)
        assert tr.exceptional() == [(c.step, c.event)], c.label
        assert ((v - E.TAU * p["a"]) % bls.R == 0) == p["valid"]
        # the bytes carry the chosen logs
        assert c.data == bls.compress(bls.mul(p["c"], bls.G1)) + p["z"].to_bytes(32, "big") + p["y"].to_bytes(32, "big") + bls.compress(bls.mul(p["a"], bls.G1))
    assert sorted(c.params["valid"] for c in cases) == [False] * 4 + [True] * 4
    trivial = [c for c in cases if c.params["a"] == 0]
    assert len(trivial) == 1 and _combine(trivial[0].params)[0] == 0 and trivial[0].params["valid"]


def test_kzg_combine_tracer_on_points():
    """over real points the combine gives C + [z] pi - [y] G, with the events of the discrete-log trace"""
    for c in E.kzg_cases()[:4]:
        p = c.params
        pts = bls.generator_multiples([p["c"], p["a"]])
        v, tr = E.run(E.kzg_combine, E.BLS_G1, pts[0], p["z"], p["y"], pts[1], bls.G1)
        vl, tl = _combine(p)
        assert v == bls.mul(vl, bls.G1) and [e for e in tr.events if e[0][0] in ("C", "-yG")] == [e for e in tl.events if e[0][0] in ("C", "-yG")]


def test_kzg_verdicts_against_the_pairing():
    """e(C - [y] G + [z] pi, G2) e(-pi, [tau] G2) = 1 in bls_pairing_ref exactly where the discrete logs say so"""
    tau_g2 = B.g2_mul(E.TAU, B.G2)
    for c in [c for c in E.kzg_cases() if c.step == ("C", 0) and c.event == E.DOUBLE]:
        p = c.params
        v, _ = _combine(p)
        pi = bls.mul(p["a"], bls.G1)
        assert B.pairing_check([(bls.mul(v, bls.G1), B.G2), (ops.G1.neg(pi), tau_g2)]) == p["valid"], c.label
