"""CPU tests: pin the C++ oracle against the pure-Python reference, the golden fixtures and the KATs the
reference itself holds (SURVEY.md section 8c).  No GPU needed."""
import os

import numpy as np
import pytest

import cpu_oracle as orc
import pyref as o

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def test_constants_match_reference_sources():
    # ALT_BN128_PRIME, /root/reference/crates/vm/levm/src/precompiles.rs:746-751 (little-endian u64 limbs)
    limbs = [0x3c208c16d87cfd47, 0x97816a916871ca8d, 0xb85045b68181585d, 0x30644e72e131a029]
    assert sum(v << (64 * i) for i, v in enumerate(limbs)) == o.P
    assert (o.R - 1) % (1 << 28) == 0 and (o.R - 1) % (1 << 29) != 0
    assert pow(o.ROOT_2_28, 1 << 28, o.R) == 1 and pow(o.ROOT_2_28, 1 << 27, o.R) == o.R - 1


def test_reference_kats_scalar_mul():
    g = o.g1_to_be(o.G1_GEN)
    # 7*(1,2): /root/reference/test/tests/l2/integration_tests.rs:572
    rc, out = orc.g1_mul_be(g, (7).to_bytes(32, "big"))
    assert rc == 0 and out.hex() == ("17072b2ed3bb8d759a5325f477629386cb6fc6ecb801bd76983a6b86abffe078"
                                     "168ada6cd130dd52017bb54bfa19377aadfe3bf05d18f41b77809f7f60d4af9e")
    rc, out = orc.g1_add_be(g, g)
    assert out.hex() == ("030644e72e131a029b85045b68181585d97816a916871ca8d3c208c16d87cfd3"
                         "15ed738c0e0a7c92e7845f96b2ae9c0a68a6a449e3538fc7ff3ebf7a5a18a2c4")
    rc, out = orc.g1_mul_be(g, o.R.to_bytes(32, "big"))
    assert rc == 1 and out == bytes(64)  # status 1 = ok-infinity (zisk.rs:144-172)


def test_reference_pairing_vector_points_decode():
    """G1/G2 points of test_ec_pairing_a (/root/reference/test/tests/levm/precompile_tests.rs:17-24) are on
    curve under the x_im|x_re|y_im|y_re order; the out-of-range point of :143-151 is rejected with status 2."""
    data = bytes.fromhex(
        "1c76476f4def4bb94541d57ebba1193381ffa7aa76ada664dd31c16024c43f593034dd2920f673e204fee2811c678745fc819b55d3e9d294e45c9b03a76aef41"
        "209dd15ebff5d46c4bd888e51a93cf99a7329636c63514396b4a452003a35bf704bf11ca01483bfa8b34b43561848d28905960114c8ac04049af4b6315a41678"
        "2bb8324af6cfc93537a2ad1a445cfd0ca2a71acd7ac41fadbf933c2a51be344d120a2a4cf30c1bf9845f20c6fe39e07ea2cce61f0c9bb048165fe5e4de877550"
        "111e129f1cf1097710d41c4ac70fcdfa5ba2023c6ff1cbeac322de49d1b6df7c2032c61a830e3c17286de9462bf242fca2883585b93870a73853face6a6bf411"
        "198e9393920d483a7260bfb731fb5d25f1aa493335a9e71297e485b7aef312c21800deef121f1e76426a00665e5c4479674322d4f75edadd46debd5cd992f6ed"
        "090689d0585ff075ec9e99ad690c3395bc4b313370b38ef355acdadcd122975b12c85ea5db8c6deb4aab71808dcb408fe3d1e7690c43d37b4ce6cc0166fa7daa")
    for off in (0, 192):
        g1, g2 = data[off:off + 64], data[off + 64:off + 192]
        assert o.g1_on_curve(o.g1_from_be(g1)) and o.g2_on_curve(o.g2_from_be(g2))
        assert orc.g1_native_to_be(orc.g1_be_to_native(g1)) == g1
        assert orc.g2_native_to_be(orc.g2_be_to_native(g2)) == g2
    assert o.g2_from_be(data[192 + 64:384]) == o.G2_GEN
    oob = (o.P + 1).to_bytes(32, "big") + (o.P + 2).to_bytes(32, "big")
    with pytest.raises(ValueError, match="status 2"):
        orc.g1_be_to_native(oob)
    with pytest.raises(ValueError, match="status 3"):
        orc.g1_be_to_native((1).to_bytes(32, "big") + (3).to_bytes(32, "big"))


def test_field_core_vs_python():
    rng = np.random.default_rng(7)
    for field, mod in (("fq", o.P), ("fr", o.R)):
        a = [int.from_bytes(rng.bytes(32), "little") % mod for _ in range(200)] + [0, 1, mod - 1]
        b = [int.from_bytes(rng.bytes(32), "little") % mod for _ in range(200)] + [mod - 1, mod - 1, mod - 1]
        got = orc.array_to_ints(orc.field_mul(field, orc.ints_to_array(a), orc.ints_to_array(b)))
        rinv = pow(o.MONT, -1, mod)
        assert got == [x * y * rinv % mod for x, y in zip(a, b)]
    x = orc.ints_to_array([5, o.R - 1, 0])
    assert orc.array_to_ints(orc.fr_to_mont(x)) == [5 * o.MONT % o.R, (o.R - 1) * o.MONT % o.R, 0]
    assert (orc.fr_from_mont(orc.fr_to_mont(x)) == x).all()


def test_rand_and_chain_generators():
    assert orc.array_to_ints(orc.rand_fr(o.SEED_SCALARS, 3, 9)) == [o.rand_fr(o.SEED_SCALARS, 3 + i) for i in range(9)]
    k, d = o.chain_scalar(o.SEED_POINTS)
    ref = o.chain_points(o._Fq, o.G1_GEN, o.SEED_POINTS, 50)
    assert orc.g1_native_to_be(orc.g1_chain(50, k, d)) == b"".join(o.g1_to_be(p) for p in ref)
    ref2 = o.chain_points(o._Fq2, o.G2_GEN, o.SEED_POINTS, 20)
    assert orc.g2_native_to_be(orc.g2_chain(20, k, d)) == b"".join(o.g2_to_be(p) for p in ref2)


def test_window_rule_is_arks():
    # ark-ec 0.5.0: c = 3 if n < 32 else ln_without_floats(n) + 2  ->  10 / 15 / 18 at 2^12 / 2^20 / 2^24
    assert [orc.lib().orc_msm_window(n) for n in (1, 31, 32, 1 << 12, 1 << 20, 1 << 24)] == [3, 3, 5, 10, 15, 18]


def test_golden_ntt_2_12():
    g = np.load(os.path.join(GOLD, "ntt_2_12.npz"))
    a = orc.fr_to_mont(g["input_canonical"])
    assert (orc.fr_from_mont(orc.fr_ntt(a, 12)) == g["forward_canonical"]).all()
    assert (orc.fr_from_mont(orc.fr_ntt(a, 12, orc.NTT_COSET)) == g["coset5_forward_canonical"]).all()
    assert (orc.fr_ntt(orc.fr_ntt(a, 12), 12, orc.NTT_INVERSE) == a).all()
    assert (orc.fr_ntt(orc.fr_ntt(a, 12, orc.NTT_COSET), 12, orc.NTT_INVERSE | orc.NTT_COSET) == a).all()
    assert (orc.fr_ntt(a, 12, threads=1) == orc.fr_ntt(a, 12, threads=4)).all()


def test_golden_msm_2_12_and_small():
    g = np.load(os.path.join(GOLD, "msm_g1_2_12.npz"))
    pts = orc.g1_be_to_native(g["points_be"].tobytes())
    for method in (0, 1):
        assert orc.g1_msm(pts, g["scalars"], method) == g["result_be"].tobytes()
    assert orc.g1_msm(pts, g["scalars"], 0, threads=1) == g["result_be"].tobytes()
    k, d = o.chain_scalar(o.SEED_POINTS)
    assert (pts == orc.g1_chain(4096, k, d)).all()
    s = np.load(os.path.join(GOLD, "msm_small.npz"))
    for m in (1, 2, 3, 31, 32, 33):
        assert orc.g1_msm(pts[:m], s[f"g1_{m}_scalars"]) == s[f"g1_{m}_result"].tobytes(), m
    p2 = orc.g2_be_to_native(s["g2_points_be"].tobytes())
    for m in (1, 2, 33):
        assert orc.g2_msm(p2[:m], s[f"g2_{m}_scalars"]) == s[f"g2_{m}_result"].tobytes(), m


def test_ntt_small_sizes_vs_definition():
    for lg in range(0, 7):
        a = orc.rand_fr(o.SEED_NTT, 0, 1 << lg)
        ai, am = orc.array_to_ints(a), orc.fr_to_mont(a)
        for fl, kw in ((0, {}), (1, dict(inverse=True)), (2, dict(coset=5)), (3, dict(inverse=True, coset=5)), (2, dict(coset=11))):
            got = orc.array_to_ints(orc.fr_from_mont(orc.fr_ntt(am, lg, fl, coset_gen=kw.get("coset"))))
            assert got == o.ntt_direct(ai, **kw), (lg, fl)


def test_msm_properties():
    """size-independent properties used at full size on the GPU: linearity and the chain closed form."""
    k, d = o.chain_scalar(o.SEED_POINTS)
    n = 3000
    pts = orc.g1_chain(n, k, d)
    s, t = orc.rand_fr(1, 0, n), orc.rand_fr(2, 0, n)
    st = orc.ints_to_array([(a + b) % o.R for a, b in zip(orc.array_to_ints(s), orc.array_to_ints(t))])
    rc, summed = orc.g1_add_be(orc.g1_msm(pts, s), orc.g1_msm(pts, t))
    assert summed == orc.g1_msm(pts, st)
    dot = orc.chain_dot(s, k, d)
    assert dot == sum(a * (k + i * d) for i, a in enumerate(orc.array_to_ints(s))) % o.R
    assert orc.g1_mul_be(o.g1_to_be(o.G1_GEN), dot.to_bytes(32, "big"))[1] == orc.g1_msm(pts, s)
    # edge distributions agree between Pippenger and the naive definition
    for vals in ([0] * 64, [1] * 64, [o.R - 1] * 64, [o.R + 3] * 64, [(1 << 256) - 1] * 64):
        sc = orc.ints_to_array(vals)
        assert orc.g1_msm(pts[:64], sc, 0) == orc.g1_msm(pts[:64], sc, 1)


def test_ntt_eval_output_is_the_definition():
    a = orc.fr_to_mont(orc.rand_fr(5, 0, 1 << 10))
    f = orc.fr_ntt(a, 10)
    for k in (0, 1, 513, 1023):
        assert (orc.fr_ntt_eval_output(a, 10, k) == f[k]).all()
    ai = orc.array_to_ints(orc.fr_from_mont(a))
    w = o.root_of_unity(10)
    assert orc.array_to_ints(orc.fr_from_mont(orc.fr_ntt_eval_output(a, 10, 3).reshape(1, 4)))[0] == sum(v * pow(w, 3 * j, o.R) for j, v in enumerate(ai)) % o.R


# ---- the reference's own BN254 KATs (tests/golden/pairing_kats.json, extracted by make_pairing_kats.py) ----
import json as _json


def _pairs(calldata: bytes):
    return [(o.g1_from_be(calldata[i:i + 64]), o.g2_from_be(calldata[i + 64:i + 192])) for i in range(0, len(calldata), 192)]


def test_reference_pairing_kats_replay_on_the_oracle_arithmetic():
    """All 14 ecpairing vectors of the reference (precompile_tests.rs:17-140): every point decodes (C++ oracle and
    pyref agree it is on the curve) and the pairing product computed with pyref's field/curve arithmetic gives the
    expected boolean.  This pins Fq, Fq2, the G1/G2 encodings and both group laws to the reference's own answers."""
    kats = _json.load(open(os.path.join(GOLD, "pairing_kats.json")))
    assert len(kats["vectors"]) == 14
    for v in kats["vectors"]:
        data = bytes.fromhex(v["calldata"])
        pairs = _pairs(data)
        for i, (g1, g2) in enumerate(pairs):
            assert o.g1_on_curve(g1) and o.g2_on_curve(g2), v["name"]
            assert orc.g1_native_to_be(orc.g1_be_to_native(data[192 * i:192 * i + 64])) == data[192 * i:192 * i + 64]
            assert orc.g2_native_to_be(orc.g2_be_to_native(data[192 * i + 64:192 * i + 192])) == data[192 * i + 64:192 * i + 192]
        assert o.pairing_check(pairs) == bool(v["expected"]), v["name"]
    oob = bytes.fromhex(kats["coordinate_out_of_bounds_calldata"])
    with pytest.raises(ValueError, match="status 2"):  # CoordinateExceedsFieldModulus (precompile_tests.rs:143-151)
        orc.g1_be_to_native(oob[:64])


def test_oracle_msm_is_bilinear_under_the_kat_pinned_pairing():
    """MSM over the reference's KAT points: e(sum s_i P_i, Q) * prod e(-P_i, s_i Q) == 1, with the C++ oracle's
    Pippenger on the left and pyref scalar multiplications on the right -- ties the MSM oracle to the pairing that
    the reference's vectors pin (the reference has no MSM vector of its own)."""
    kats = _json.load(open(os.path.join(GOLD, "pairing_kats.json")))
    g1s = []
    for v in kats["vectors"][:5]:
        g1s += [p for p, _ in _pairs(bytes.fromhex(v["calldata"])) if p is not None]
    g1s = g1s[:8]
    scalars = [o.rand_fr(77, i) for i in range(len(g1s))]
    pts_native = orc.g1_be_to_native(b"".join(o.g1_to_be(p) for p in g1s))
    a = o.g1_from_be(orc.g1_msm(pts_native, orc.ints_to_array(scalars)))
    q = o.G2_GEN
    check = [(a, q)] + [(o.pt_neg(o._Fq, p), o.g2_mul(s, q)) for p, s in zip(g1s, scalars)]
    assert o.pairing_check(check)
    # and the G2 side: e(P, sum s_i Q_i) with Q_i = i-th multiples of the KAT G2 generator
    g2s = [o.g2_mul(i + 2, q) for i in range(4)]
    b = o.g2_from_be(orc.g2_msm(orc.g2_be_to_native(b"".join(o.g2_to_be(x) for x in g2s)), orc.ints_to_array(scalars[:4])))
    pneg = o.pt_neg(o._Fq, o.G1_GEN)
    assert o.pairing_check([(o.G1_GEN, b)] + [(o.g1_mul(s, pneg), x) for s, x in zip(scalars[:4], g2s)])


def test_tower_pairing_restatement_agrees_with_the_kats_and_with_pyref():
    """oracle/pyref_tower.py (plain ate, Fq2/Fq6/Fq12 tower -- the algorithm of ethrex_b200/csrc/pairing.cu) gives
    the reference's expected answer on all 14 ecpairing vectors, i.e. the same answers as pyref's independent
    optimal-ate statement."""
    import pyref_tower as tw
    kats = _json.load(open(os.path.join(GOLD, "pairing_kats.json")))
    for v in kats["vectors"]:
        pairs = _pairs(bytes.fromhex(v["calldata"]))
        assert tw.pairing_check(pairs) == bool(v["expected"]), v["name"]
    # bilinearity on fresh points: e(aP, bQ) * e(-abP, Q) == 1, and a wrong product is not 1
    a, b = 0x1234567, 0x89abcdef01
    P1, Q1 = o.g1_mul(a, o.G1_GEN), o.g2_mul(b, o.G2_GEN)
    neg = o.g1_mul(o.R - (a * b) % o.R, o.G1_GEN)
    assert tw.pairing_check([(P1, Q1), (neg, o.G2_GEN)])
    assert not tw.pairing_check([(P1, Q1), (o.g1_mul(o.R - (a * b + 1) % o.R, o.G1_GEN), o.G2_GEN)])


def test_toy_groth16_instance_is_sound_under_the_kat_pinned_pairing():
    """tests/groth16_toy.py (the real small Groth16 instance the GPU prover is checked against): the proof computed in
    the exponent satisfies the verification equation under the pairing the reference's KATs pin; a wrong public input
    or a perturbed proof does not."""
    import pyref_tower as tw
    from groth16_toy import ToyGroth16
    toy = ToyGroth16(3)
    x = 0x1234567
    z = toy.assign(x)
    proof = toy.expected_proof(z)
    assert tw.pairing_check(_pairs(toy.verifier_calldata(proof, x)))
    assert not tw.pairing_check(_pairs(toy.verifier_calldata(proof, x + 1)))
    bad = proof[:192] + o.g1_to_be(o.g1_add(o.g1_from_be(proof[192:256]), o.G1_GEN))
    assert not tw.pairing_check(_pairs(toy.verifier_calldata(bad, x)))


def test_groth16_golden_fixture_is_current():
    """tests/golden/groth16_toy.json matches what the toy instance produces today, and its verifier calldata passes the
    tower pairing (the GPU side of the same fixture: test_gpu_parity.py::test_groth16_golden_fixture)."""
    import pyref_tower as tw
    from groth16_toy import ToyGroth16
    gold = _json.load(open(os.path.join(GOLD, "groth16_toy.json")))
    inst = gold["instances"][0]
    toy = ToyGroth16(inst["log_n"])
    for case in inst["cases"]:
        x = int(case["public_input"], 16)
        proof = toy.expected_proof(toy.assign(x))
        assert proof.hex() == case["proof"] and toy.verifier_calldata(proof, x).hex() == case["verifier_calldata"]
    assert tw.pairing_check(_pairs(bytes.fromhex(inst["cases"][0]["verifier_calldata"])))


def test_ntt_root_presets_in_the_library_are_the_published_generators():
    """b200zk_ntt_root_preset (no device needed): preset 0 = ark-poly / gnark-crypto 5^((r-1)/2^28), preset 1 =
    halo2curves 7^((r-1)/2^28) -- the value SURVEY.md section 8c records -- and the oracle's NTT accepts either."""
    import ctypes
    from ethrex_b200 import _ffi
    buf = ctypes.create_string_buffer(32)
    assert _ffi.lib.b200zk_ntt_root_preset(0, buf) == 0 and int.from_bytes(buf.raw, "little") == o.ROOT_2_28 == pow(5, (o.R - 1) >> 28, o.R)
    halo2 = pow(7, (o.R - 1) >> 28, o.R)
    assert _ffi.lib.b200zk_ntt_root_preset(1, buf) == 0 and int.from_bytes(buf.raw, "little") == halo2
    assert halo2 == 0x03ddb9f5166d18b798865ea93dd31f743215cf6dd39329c8d34f1ed960c37c9c
    assert pow(halo2, 1 << 28, o.R) == 1 and pow(halo2, 1 << 27, o.R) == o.R - 1
    assert _ffi.lib.b200zk_ntt_root_preset(2, buf) == _ffi.ERR_INVALID_ARG
    # the C++ oracle under halo2's root = the definition sum_j a_j w^(jk) with w = halo2^(2^(28-k))
    import cpu_oracle as orc
    n, log_n = 8, 3
    a = [3, 1, 4, 1, 5, 9, 2, 6]
    w = pow(halo2, 1 << (28 - log_n), o.R)
    want = [sum(a[j] * pow(w, j * k, o.R) for j in range(n)) % o.R for k in range(n)]
    got = orc.array_to_ints(orc.fr_from_mont(orc.fr_ntt(orc.fr_to_mont(orc.ints_to_array(a)), log_n, 0, root_2_28=halo2)))
    assert got == want


def test_bls12_381_oracle_constants():
    """oracle/bls_ref.py against the public constants of the curve: generator on the curve and of order r, its compressed
    form, the identity's form, the 4096-th root of unity, the Lagrange basis summing to one -- and the product's host-side
    KZG bookkeeping (ethrex_b200/kzg.py) agreeing with it on the domain."""
    import bls_ref as b
    from ethrex_b200 import kzg
    assert b.on_curve(b.G1) and b.mul(b.R, b.G1) is None
    assert b.compress(b.G1) == b.G1_COMPRESSED and b.decompress(b.G1_COMPRESSED) == b.G1
    assert b.compress(None) == bytes([0xC0]) + bytes(47) and b.decompress(b.compress(None)) is None
    neg = (b.G1[0], b.P - b.G1[1])
    assert b.compress(neg)[0] & 0x20 != b.compress(b.G1)[0] & 0x20 and b.decompress(b.compress(neg)) == neg
    assert pow(b.ROOT_4096, 4096, b.R) == 1 and pow(b.ROOT_4096, 2048, b.R) == b.R - 1
    assert kzg.BLS_MODULUS == b.R and kzg.roots_of_unity_brp()[1] == pow(b.ROOT_4096, 2048, b.R)  # brp(1) = 2048
    lag = b.lagrange_setup_scalars(987654321, 16)
    assert sum(lag) % b.R == 1
    assert b.generator_multiples([5, 0, b.R - 1]) == [b.mul(5, b.G1), None, b.mul(b.R - 1, b.G1)]
    # Fiat-Shamir challenge: domain | degree | blob | commitment, reduced mod r
    blob, c = bytes(4096 * 32), b.compress(None)
    import hashlib
    want = int.from_bytes(hashlib.sha256(b"FSBLOBVERIFY_V1_" + (4096).to_bytes(16, "big") + blob + c).digest(), "big") % b.R
    assert kzg.KzgSettings.compute_challenge(blob, c) == want


def _bls_chain_points(raw: bytes):
    import bls_ref as b
    pts = []
    for i in range(len(raw) // 96):
        x, y = int.from_bytes(raw[96 * i:96 * i + 48], "big"), int.from_bytes(raw[96 * i + 48:96 * i + 96], "big")
        pts.append(None if raw[96 * i] == 0x40 else (x, y))
    return pts


def test_bls12_381_chain_is_the_generator_multiples():
    """bls_ref.chain -- the synthetic BLS12-381 bases whose MSM has a closed form -- against generator_multiples: sampled
    indices across block boundaries, every point on the curve, and chains that pass through the identity and through a
    doubling (k = 0: P_1 = D, then P_1 + D = 2D)."""
    import bls_ref as b
    k, d = 0x1234567890ABCDEF1234567890ABCDEF % b.R, 0xFEDCBA0987654321FEDCBA0987654321 % b.R
    n = 5000
    raw = b.chain(n, k, d)
    assert len(raw) == 96 * n
    pts = _bls_chain_points(raw)
    assert all(b.on_curve(p) and p is not None for p in pts)
    idx = [0, 1, 2, 4095, 4096, 4097, n - 1]
    assert [pts[i] for i in idx] == b.generator_multiples([k + i * d for i in idx])
    # small blocks: every block boundary; k + 3d = 0 puts the identity at index 3; k = 0 starts at the identity
    for kk, dd in (((b.R - 3 * d) % b.R, d), (0, d), (k, 0)):
        pts = _bls_chain_points(b.chain(9, kk, dd, block=4))
        assert pts == b.generator_multiples([kk + i * dd for i in range(9)]), (kk, dd)
    assert _bls_chain_points(b.chain(9, (b.R - 3 * d) % b.R, d))[3] is None
