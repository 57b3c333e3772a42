"""CPU checks of the BLS12-381 pairing and KZG verification: the independent oracle (tests/bls_pairing_ref.py) against the
reference's EIP-2537 vectors and bilinearity, G2 compression, the final exponentiation's x-chain identity, every constant
of ethrex_b200/csrc/bls_pairing.cu recomputed from its definition, a Python verifier over the known-tau setup, and the
ptxas report of the new kernels."""
import json
import os
import re

import pytest

import bls_pairing_ref as B
import bls_ref as bls

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "ethrex_b200", "csrc")
P, R = B.P, B.R
X = -B.X_ABS


def _pairs(calldata: bytes):
    return [(B.g1_from_eip2537(calldata[i:i + 128]), B.g2_from_eip2537(calldata[i + 128:i + 384])) for i in range(0, len(calldata), 384)]


def test_oracle_reference_vectors():
    kats = json.load(open(os.path.join(HERE, "golden", "bls12_pairing_kats.json")))["vectors"]
    assert [int(B.pairing_check(_pairs(bytes.fromhex(v["calldata"])))) for v in kats] == [v["expected"] for v in kats] == [0, 0, 1]


@pytest.mark.parametrize("a,b", [(2, 3), (R - 1, 5), (0x1234567890ABCDEF, 0xFEDCBA987654321)])
def test_oracle_bilinearity(a, b):
    lhs = B.pairing(bls.mul(a, B.G1), B.g2_mul(b, B.G2))
    assert lhs == B.f12_pow(B.pairing(B.G1, B.G2), a * b % R)
    assert B.pairing_check([(bls.mul(a, B.G1), B.g2_mul(b, B.G2)), (bls.mul(a * b, B.G1), B.g2_neg(B.G2))])


def test_g2_compression_round_trip():
    assert B.g2_compress(B.G2) == B.G2_COMPRESSED and B.g2_decompress(B.G2_COMPRESSED) == B.G2
    assert B.g2_decompress(B.g2_compress(None)) is None
    for k in (1, 2, 3, R - 1, 0xABCDEF):
        q = B.g2_mul(k, B.G2)
        assert B.g2_on_curve(q) and B.g2_decompress(B.g2_compress(q)) == q
    assert B.g2_in_subgroup(B.G2) and not B.g2_in_subgroup(B.g2_random_point(1))
    with pytest.raises(ValueError):
        B.g2_decompress(B.G2_COMPRESSED[:48] + P.to_bytes(48, "big"))


def test_fp2_sqrt_algorithm_of_the_device():
    """bls12.cuh Fp2_381::sqrt_candidate, restated: a1 = a^((p-3)/4), alpha = a1^2 a, x0 = a1 a; u x0 if alpha = -1,
    else (1 + alpha)^((p-1)/2) x0"""
    for seed in range(1, 40):
        a = ((seed * 0x9E3779B97F4A7C15) % P, (seed * 0x632BE59BD9B4E019 + 7) % P)
        a1 = B.f2_pow(a, (P - 3) // 4)
        x0 = B.f2_mul(a1, a)
        alpha = B.f2_mul(a1, x0)
        x = (-x0[1] % P, x0[0]) if alpha == (P - 1, 0) else B.f2_mul(B.f2_pow(B.f2_add((1, 0), alpha), (P - 1) // 2), x0)
        assert (B.f2_sqr(x) == a) == (B.f2_sqrt(a) is not None), seed


def test_final_exponentiation_x_chain():
    assert (P ** 4 - P ** 2 + 1) % R == 0
    assert (X - 1) ** 2 * (X + P) * (X * X + P * P - 1) + 3 == 3 * (P ** 4 - P ** 2 + 1) // R
    assert (P ** 12 - 1) % R == 0 and (P ** 6 - 1) * (P ** 2 + 1) * (P ** 4 - P ** 2 + 1) == P ** 12 - 1
    assert R % 3 != 0  # cubing is a bijection on the order-r group: z^3 = 1 iff z = 1
    assert bin(B.X_ABS).count("1") - 1 == 5 and B.X_ABS.bit_length() == 64  # 63 doublings + 5 additions = 68 lines


def _limbs(words):
    return sum(int(w, 16) << (32 * i) for i, w in enumerate(words))


def test_constants_of_the_source():
    src = open(os.path.join(CSRC, "bls_pairing.cu")).read()

    def block(name):
        body = re.search(name + r"[^=]*= \{(.*?)\};", src, re.S).group(1)
        return re.findall(r"0x([0-9a-f]+)u", body)
    xi = (1, 1)
    f1 = block("kFrob1")
    assert len(f1) == 6 * 2 * 12
    for k in range(6):
        want = B.f2_pow(xi, k * (P - 1) // 6)
        assert (_limbs(f1[24 * k:24 * k + 12]), _limbs(f1[24 * k + 12:24 * k + 24])) == want, k
    f2 = block("kFrob2")
    for k in range(6):
        assert (_limbs(f2[12 * k:12 * k + 12]), 0) == B.f2_pow(xi, k * (P * P - 1) // 6), k
    g = block("kG1Gen")
    assert (_limbs(g[:12]), _limbs(g[12:])) == bls.G1
    g2 = re.search(r"kG2GenCompressed\[96\] = \{(.*?)\};", src, re.S).group(1)
    assert bytes(int(b, 16) for b in re.findall(r"0x([0-9a-f]{2})", g2)) == B.G2_COMPRESSED
    assert re.search(r"kX = 0x([0-9a-f]+)ull", src).group(1) == format(B.X_ABS, "x")
    assert re.search(r"kLines = (\d+);", src).group(1) == "68"


TAU = 0x2F1B7C93D4A5E6F708192A3B4C5D6E7F8091A2B3C4D5E6F708192A3B4C5D6E7F % R


def _verify(commitment, z, y, proof, tau_g2):
    """the device's rewrite of c-kzg verify_kzg_proof: e(C - [y]G1 + [z]pi, G2) e(-pi, [tau]G2) == 1"""
    c, pi = bls.decompress(commitment), bls.decompress(proof)
    lhs = bls.add(bls.add(c, bls.mul(-y % R, B.G1)), bls.mul(z, pi))
    return B.pairing_check([(lhs, B.G2), (None if pi is None else (pi[0], P - pi[1]), tau_g2)])


def test_python_verifier_over_the_known_tau_setup():
    """p(X) = 3 + 5X + 7X^2: C = [p(tau)], proof at z = [(p(tau) - y)/(tau - z)] -- accepted; tampered -- rejected"""
    def p(x):
        return (3 + 5 * x + 7 * x * x) % R
    z = 0x123456789
    y = p(z)
    c = bls.compress(bls.mul(p(TAU), B.G1))
    proof = bls.compress(bls.mul((p(TAU) - y) * pow(TAU - z, -1, R), B.G1))
    tau_g2 = B.g2_mul(TAU, B.G2)
    assert _verify(c, z, y, proof, tau_g2)
    assert not _verify(c, z, y + 1, proof, tau_g2)
    assert not _verify(c, z + 1, y, proof, tau_g2)
    assert not _verify(c, z, y, bls.compress(B.G1), tau_g2)
    assert not _verify(c, z, y, proof, B.g2_mul(TAU + 1, B.G2))


@pytest.mark.parametrize("kernel", ["bls_pair_decode", "bls_g2_decode", "bls_g2_prepare", "bls_miller", "pairing_check",
                                    "bls_g1_decode_subgroup", "kzg_verify_combine", "kzg_blob_terms", "kzg_blob_fold"])
def test_ptxas_lists_the_new_kernels(kernel):
    log = os.path.join(CSRC, "build", "bls_pairing.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("bls_pairing.ptxas.log not built")
    m = re.search(r"Function properties for \w*" + kernel + r"\w*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n"
                  r"ptxas info\s*: Used (\d+) registers", open(log).read())
    assert m, f"no ptxas report for {kernel}"
