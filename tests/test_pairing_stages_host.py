"""CPU checks of tests/pairing_stages_ref.py, the Python restatement the device pairing stages are compared with: each
stage against an anchor that does not share its algorithm, so the restatement is not only checked against itself.

- the tower <-> flat conversion: products agree with the schoolbook tower of field_conformance_ref;
- FROB(a) = a^p and FROB2(a) = a^(p^2) for any a;
- EXP_X(c) = c^x (x < 0) for cyclotomic c;
- the BLS x-chain final exponentiation = f^(3 (p^12 - 1)/r) exactly, the BN one = f^((p^12 - 1)/r), for any f != 0; both
  map 0 to 0, as the device's inv(0) = 0 makes them;
- after G2 preparation, T's affine point is [|x|]Q;
- the restated BLS pairing is the inverse cube of bls_pairing_ref.pairing, which shares no code with it, and bilinear;
- the cofactor factorisations, and the order of every cofactor-component point the GPU tests use."""
import random

import pytest

import bls_pairing_ref as B
import bls_ref as bls
import field_conformance_ref as ref
import pairing_stages_ref as S
import pyref
import pyref_tower as BT

P, R = S.P, S.R


def _rand(rng):
    return S._tower([(rng.randrange(P), rng.randrange(P)) for _ in range(6)])


def test_tower_layout():
    rng = random.Random(1)
    T = ref.BLS_FP12
    for _ in range(8):
        a, b = _rand(rng), _rand(rng)
        assert S.from_flat(S.to_flat(a)) == a
        assert S.mul(a, b) == T.mul(a, b)
        assert S.mul(a, S.inv(a)) == S.ONE
    assert S.mul(S.W, S.W) == ((B.f2_sqr((0, 0)), (1, 0), (0, 0)), ((0, 0),) * 3)  # w^2 = v
    assert S.power(S.W, 6) == S._tower([S.XI] + [(0, 0)] * 5)  # w^6 = 1 + u
    assert S.inv(S.ZERO) == S.ZERO


def test_frobenius_is_the_p_power():
    rng = random.Random(2)
    for a in [S.W, S._tower([(3, 7)] * 6)] + [_rand(rng) for _ in range(3)]:
        assert S.frob(a) == S.power(a, P)
        assert S.frob2(a) == S.power(a, P * P)


def test_exp_x_on_the_cyclotomic_subgroup():
    rng = random.Random(3)
    for _ in range(3):
        f = _rand(rng)
        c = S.power(f, (P ** 6 - 1) * (P * P + 1))
        assert S.mul(c, S.conj(c)) == S.ONE  # cyclotomic: conj is the inverse
        assert S.exp_x(c) == S.power(S.inv(c), S.X_ABS)
        assert S.exp_x(f) != S.power(S.inv(f), S.X_ABS)  # off the subgroup the device value is conj(f^|x|), not f^x


def test_bls_final_exponentiation_is_the_generic_power():
    rng = random.Random(4)
    lines = S.g2_prepare(B.G2)[0]
    fs = [S.W, S.conj(S.ONE), S._tower([(P - 1, 0)] + [(0, 0)] * 5), S.miller(lines, B.G1)] + [_rand(rng) for _ in range(4)]
    for f in fs:
        assert S.final_exponentiate(f) == S.power(f, S.FINAL_EXP_BLS)
    assert S.final_exponentiate(S._tower([(5, 9), (0, 0), (1, 0), (0, 0), (0, 2), (0, 0)])) == S.ONE  # Fp6: even powers of w only
    assert S.final_exponentiate(S.ZERO) == S.ZERO


def test_bn_final_exponentiation_is_the_generic_power():
    rng = random.Random(5)
    p = pyref.P
    for _ in range(4):
        f = tuple(tuple((rng.randrange(p), rng.randrange(p)) for _ in range(3)) for _ in range(2))
        assert BT.final_exponentiate(f) == BT.f12_pow(f, (p ** 12 - 1) // pyref.R)


@pytest.mark.parametrize("k", [1, 2, R - 1, 0xC0FFEE])
def test_g2_prepare_ends_at_x_times_q(k):
    q = B.g2_mul(k, B.G2)
    lines, T = S.g2_prepare(q)
    zi = B.f2_inv(T[2])
    assert (B.f2_mul(T[0], zi), B.f2_mul(T[1], zi)) == B.g2_mul(S.X_ABS, q, reduce=False)
    assert len(lines) == 68


def test_lines_vanish_at_their_points():
    """the doubling line is the tangent at T and the addition line passes through T and Q: evaluated in the untwisted
    coordinates of T itself, l = c0 + c1 x w^2 + c2 y w^3 (w^2 = v, w^3 = v w) is zero"""
    q = B.g2_mul(7, B.G2)
    for T in [(q[0], q[1], (1, 0)), (B.f2_mul(q[0], (3, 4)), B.f2_mul(q[1], (3, 4)), (3, 4))]:
        zi = B.f2_inv(T[2])
        x, y = B.f2_mul(T[0], zi), B.f2_mul(T[1], zi)
        _, (c0, c1, c2) = S.line_double(T)
        assert B.f2_add(c0, B.f2_add(B.f2_mul(c1, x), B.f2_mul(c2, y))) == (0, 0)
        _, (c0, c1, c2) = S.line_add(T, q)
        assert B.f2_add(c0, B.f2_add(B.f2_mul(c1, x), B.f2_mul(c2, y))) == (0, 0)


def test_bls_pair_is_the_inverse_cube_of_the_independent_pairing():
    e = S.pair(B.G1, B.G2)
    assert e == S.inv(S.power(S.from_flat(B.pairing(B.G1, B.G2)), 3))
    a, b = 0x1234567890ABCDEF, 0xFEDCBA987654321
    assert S.pair(bls.mul(a, B.G1), B.g2_mul(b, B.G2)) == S.power(e, a * b % R)


def test_bn_pair_is_bilinear():
    a, b = 0xABCDEF12345, 0x987654321
    g1, g2 = pyref.G1_GEN, pyref.G2_GEN
    e = BT.final_exponentiate(BT.miller_ate(g2, g1))
    assert e != BT.F12_ONE
    assert BT.final_exponentiate(BT.miller_ate(pyref.g2_mul(b, g2), pyref.g1_mul(a, g1))) == BT.f12_pow(e, a * b % pyref.R)


def test_cofactors():
    assert S.BLS_G1.factors == {3: 1, 11: 2, 10177: 2, 859267: 2, 52437899: 2}
    h2 = S.BLS_G2.factors
    assert hex(S.BLS_H2).startswith("0x5d543a95") and hex(S.BLS_H2).endswith("c7238e5")
    assert {ell: e for ell, e in h2.items() if ell < 1 << 64} == {13: 2, 23: 2, 2713: 1, 11953: 1, 262069: 1}
    assert [ell.bit_length() for ell in h2 if ell > 1 << 64] == [448]
    assert S.BN_H2 == 2 * pyref.P - pyref.R
    bn = S.BN_G2.factors
    assert {ell for ell in bn if ell < 1 << 64} == {10069, 5864401, 1875725156269} and [ell.bit_length() for ell in bn if ell > 1 << 64] == [178]


@pytest.mark.parametrize("G", [S.BLS_G1, S.BLS_G2, S.BN_G2], ids=lambda G: G.name)
def test_cofactor_component_points(G):
    """every prime of h has a point of order exactly l; the sums with a subgroup point leave the subgroup; the subgroup
    points are in it"""
    cs = G.cases()
    names = {name for name, _, _ in cs}
    assert all(f"T_{ell}" in names and f"G+T_{ell}" in names for ell in G.factors)
    for name, pt, sub in cs:
        assert G.on_curve(pt)
        assert (G.mul(G.r, pt) is None) == sub, name
    for ell in G.factors:
        t = dict((n, p) for n, p, _ in cs)[f"T_{ell}"]
        assert G.order_is(t, ell)
