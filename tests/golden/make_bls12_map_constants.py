"""Checks the map-to-curve constants of tests/bls12_map_ref.py against the curves and prints the tables bls_map.cu embeds.

    python tests/golden/make_bls12_map_constants.py        (pure Python, a few seconds; no input files but the KAT)

G1 (RFC 9380 Appendix E.2, typed from the RFC) is validated four ways; a mistyped digit in any of the 53 isogeny
coefficients breaks check 2:
  1. #E'(Fp) = #E(Fp) = p - z: [p - z] Q = O for random points Q of E' (the isogeny class of E).
  2. iso_map sends random points of E' onto E: y^2 = x^3 + 4.
  3. iso_map is a group homomorphism: iso(P + Q) = iso(P) + iso(Q).
  4. Z = 11 is what the RFC's find_z_sswu (Appendix H.2) returns: the first of 1, -1, 2, -2, ... that is a non-square,
     not -1, makes g(x) - Z irreducible and g(B'/(Z A')) a square.
G2 (Appendix E.3) is re-derived, not just checked: the 3-isogeny of E2' is Velu's, from the one root in Fp2 of E2''s
3-division polynomial, followed by one of the six isomorphisms (x, y) -> (s^2 x, s^3 y) onto E2: y^2 = x^3 + 4(1 + i).
Exactly one of the six maps (0, 0) to the reference's FP2_ZERO_MAPPED_TO_G2 (tests/golden/bls12_map_kats.json) through
SSWU and clear_cofactor by h_eff; that one must equal the oracle's table.

The printed tables are canonical little-endian 32-bit limbs; tests/test_bls12_map_host.py checks that bls_map.cu holds
exactly these."""
import json
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
for _p in (os.path.dirname(HERE), os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import bls12_map_ref as M  # noqa: E402
import bls_pairing_ref as B  # noqa: E402
import bls_ref as bls  # noqa: E402

P = M.P
Fp, Fp2 = M.Fp, M.Fp2


# ---- affine group law on y^2 = x^3 + A x + B (None = identity); E' has A != 0, so bls_ref's a = 0 law does not apply
def ec_add(F, A, p, q):
    if p is None:
        return q
    if q is None:
        return p
    (x1, y1), (x2, y2) = p, q
    if x1 == x2:
        if F.add(y1, y2) == F.zero:
            return None
        xx = F.mul(x1, x1)
        lam = F.mul(F.add(F.add(F.add(xx, xx), xx), A), F.inv0(F.add(y1, y1)))
    else:
        lam = F.mul(F.sub(y2, y1), F.inv0(F.sub(x2, x1)))
    x3 = F.sub(F.sub(F.mul(lam, lam), x1), x2)
    return x3, F.sub(F.mul(lam, F.sub(x1, x3)), y1)


def ec_mul(F, A, k, p):
    acc = None
    while k:
        if k & 1:
            acc = ec_add(F, A, acc, p)
        p = ec_add(F, A, p, p)
        k >>= 1
    return acc


def rhs(F, A, Bc, x):
    return F.add(F.mul(F.add(F.mul(x, x), A), x), Bc)


def random_point(F, A, Bc, rng):
    while True:
        x = rng.randrange(P) if F is Fp else (rng.randrange(P), rng.randrange(P))
        y = F.sqrt(rhs(F, A, Bc, x))
        if y is not None:
            return x, y


# ---- G1 checks
def check_g1_point_count(n=3, seed=1):
    rng = random.Random(seed)
    order = P + M.Z_ABS  # p - z, z = -|z|
    for _ in range(n):
        q = random_point(Fp, M.G1_A, M.G1_B, rng)
        assert ec_mul(Fp, M.G1_A, order, q) is None, "#E' != p - z"


def check_g1_iso_on_curve(n=8, seed=2):
    rng = random.Random(seed)
    for _ in range(n):
        assert bls.on_curve(M.iso_map(Fp, M.G1_TABLES, random_point(Fp, M.G1_A, M.G1_B, rng))), "iso_map leaves E"


def check_g1_iso_additive(n=4, seed=3):
    rng = random.Random(seed)
    for _ in range(n):
        p, q = random_point(Fp, M.G1_A, M.G1_B, rng), random_point(Fp, M.G1_A, M.G1_B, rng)
        iso = lambda t: M.iso_map(Fp, M.G1_TABLES, t)  # noqa: E731
        assert iso(ec_add(Fp, M.G1_A, p, q)) == bls.add(iso(p), iso(q)), "iso_map is not additive"


def _poly_mulmod(a, b, m):
    """a b mod m over Fp, lists in ascending powers, m monic"""
    r = [0] * (len(a) + len(b) - 1)
    for i, x in enumerate(a):
        for j, y in enumerate(b):
            r[i + j] += x * y
    for k in range(len(r) - 1, len(m) - 2, -1):
        c = r[k] % P
        if c:
            for j in range(len(m)):
                r[k - len(m) + 1 + j] -= c * m[j]
    return [c % P for c in r[:len(m) - 1]]


def _has_root(cubic):
    """whether the monic cubic has a root in Fp: x^p = x somewhere, i.e. gcd(x^p - x, cubic) != 1"""
    acc, base = [1, 0, 0], [0, 1, 0]
    for bit in bin(P)[2:]:
        acc = _poly_mulmod(acc, acc, cubic)
        if bit == "1":
            acc = _poly_mulmod(acc, base, cubic)
    a, b = cubic, [(acc[0]) % P, (acc[1] - 1) % P, acc[2]]  # x^p - x mod cubic
    while any(b):
        while b and b[-1] == 0:
            b = b[:-1]
        inv = pow(b[-1], -1, P)
        a = a[:]
        while len(a) >= len(b):
            c = a[-1] * inv % P
            d = len(a) - len(b)
            for j, y in enumerate(b):
                a[d + j] = (a[d + j] - c * y) % P
            while a and a[-1] == 0:
                a = a[:-1]
        a, b = b, a
        if not b:
            break
    return len(a) > 1


def find_z_sswu_g1():
    """RFC 9380 Appendix H.2 over Fp with the G1 curve E'"""
    is_square = lambda v: pow(v, (P - 1) // 2, P) in (0, 1)  # noqa: E731
    ctr = 1
    while True:
        for z in (ctr, -ctr % P):
            if is_square(z) or z == P - 1:
                continue
            if _has_root([(M.G1_B - z) % P, M.G1_A, 0, 1]):
                continue
            if is_square(rhs(Fp, M.G1_A, M.G1_B, M.G1_B * pow(z * M.G1_A, -1, P) % P)):
                return z
        ctr += 1


# ---- G2 derivation: Fp2 polynomials as ascending lists of pairs
def _p2_trim(a):
    while a and a[-1] == (0, 0):
        a = a[:-1]
    return a


def _p2_mulmod(a, b, m):
    r = [(0, 0)] * (len(a) + len(b) - 1)
    for i, x in enumerate(a):
        for j, y in enumerate(b):
            r[i + j] = B.f2_add(r[i + j], B.f2_mul(x, y))
    return _p2_mod(r, m)


def _p2_mod(a, m):
    a, inv = _p2_trim(list(a)), B.f2_inv(m[-1])
    while len(a) >= len(m):
        c, d = B.f2_mul(a[-1], inv), len(a) - len(m)
        for j, y in enumerate(m):
            a[d + j] = B.f2_sub(a[d + j], B.f2_mul(c, y))
        a = _p2_trim(a)
    return a


def _p2_powmod(a, e, m):
    acc = [(1, 0)]
    for bit in bin(e)[2:]:
        acc = _p2_mulmod(acc, acc, m)
        if bit == "1":
            acc = _p2_mulmod(acc, a, m)
    return acc


def _p2_gcd(a, b):
    a, b = _p2_trim(a), _p2_trim(b)
    while b:
        a, b = b, _p2_mod(a, b)
    inv = B.f2_inv(a[-1])
    return [B.f2_mul(c, inv) for c in a]


def _p2_sub(a, b):
    n = max(len(a), len(b))
    a, b = a + [(0, 0)] * (n - len(a)), b + [(0, 0)] * (n - len(b))
    return _p2_trim([B.f2_sub(x, y) for x, y in zip(a, b)])


def _p2_roots(f, rng):
    """the roots in Fp2 of f (Cantor-Zassenhaus)"""
    g = _p2_gcd(f, _p2_sub(_p2_powmod([(0, 0), (1, 0)], P * P, f), [(0, 0), (1, 0)]))
    out, todo = [], [g]
    while todo:
        h = todo.pop()
        if len(h) == 1:
            continue
        if len(h) == 2:
            out.append(B.f2_neg(h[0]))
            continue
        d = (rng.randrange(P), rng.randrange(P))
        s = _p2_gcd(h, _p2_sub(_p2_powmod([d, (1, 0)], (P * P - 1) // 2, h), [(1, 0)]))
        if 1 < len(s) < len(h):
            q = h
            # h / s by long division
            quo = [(0, 0)] * (len(q) - len(s) + 1)
            q = list(q)
            while len(q) >= len(s):
                c, k = q[-1], len(q) - len(s)
                quo[k] = c
                for j, y in enumerate(s):
                    q[k + j] = B.f2_sub(q[k + j], B.f2_mul(c, y))
                q = _p2_trim(q)
            todo += [s, quo]
        else:
            todo.append(h)
    return out


def derive_g2_isogeny(expected_zero_image: bytes, seed=4):
    """Velu's 3-isogeny out of E2', composed with the isomorphism onto E2 that maps (0, 0) to the reference's vector"""
    rng = random.Random(seed)
    a, b = M.G2_A, M.G2_B
    f2 = B.f2_mul
    # 3-division polynomial 3 x^4 + 6 a x^2 + 12 b x - a^2
    psi3 = [B.f2_neg(f2(a, a)), f2((12, 0), b), f2((6, 0), a), (0, 0), (3, 0)]
    roots = _p2_roots(psi3, rng)
    assert len(roots) == 1, "E2' should have one Fp2-rational 3-kernel"
    x0 = roots[0]
    vq = B.f2_add(f2((6, 0), f2(x0, x0)), f2((2, 0), a))
    uq = f2((4, 0), rhs(Fp2, a, b, x0))
    a2 = B.f2_sub(a, f2((5, 0), vq))
    b2 = B.f2_sub(b, f2((7, 0), B.f2_add(uq, f2(x0, vq))))
    assert a2 == (0, 0), "the image of E2' has j = 0"
    # X = [x (x - x0)^2 + vq (x - x0) + uq] / (x - x0)^2,  Y = y [(x - x0)^3 - vq (x - x0) - 2 uq] / (x - x0)^3
    n0 = B.f2_neg(x0)
    d2 = [f2(x0, x0), f2((2, 0), n0), (1, 0)]
    d3 = [f2(n0, f2(x0, x0)), f2((3, 0), f2(x0, x0)), f2((3, 0), n0), (1, 0)]
    xnum = [B.f2_add(uq, f2(vq, n0)), B.f2_add(d2[0], vq), d2[1], (1, 0)]
    ynum = [B.f2_sub(B.f2_sub(d3[0], f2(vq, n0)), f2((2, 0), uq)), B.f2_sub(d3[1], vq), d3[2], (1, 0)]
    # (x, y) -> (s^2 x, s^3 y) with s^6 b2 = 4 (1 + i)
    t = f2((4, 4), B.f2_inv(b2))
    found = []
    for s2 in _p2_roots([B.f2_neg(t), (0, 0), (0, 0), (1, 0)], rng):
        s = B.f2_sqrt(s2)
        if s is None:
            continue
        for sg in (s, B.f2_neg(s)):
            s3 = f2(sg, s2)
            tables = ([f2(s2, c) for c in xnum], d2[:2], [f2(s3, c) for c in ynum], d3[:3])
            q = M.iso_map(Fp2, tables, M.sswu(Fp2, a, b, M.G2_Z, (0, 0)))
            if B.g2_eip2537(M.clear_cofactor_g2_scalar(q)) == expected_zero_image:
                found.append(tables)
    assert len(found) == 1, f"{len(found)} isomorphisms reproduce the vector"
    return found[0]


def check_g2_against_vector():
    kat = json.load(open(os.path.join(HERE, "bls12_map_kats.json")))["vectors"][0]
    derived = derive_g2_isogeny(bytes.fromhex(kat["expected"]))
    assert derived == M.G2_TABLES, "the oracle's E.3 table differs from the derived isogeny"
    return derived


# ---- the tables bls_map.cu embeds
def limbs(v):
    return [(v >> (32 * k)) & 0xFFFFFFFF for k in range(12)]


def tables():
    """name -> list of field elements (G1: ints, G2: pairs), in the order bls_map.cu lays them out"""
    g1_c = [M.G1_A, M.G1_B, M.G1_Z, -M.G1_B * pow(M.G1_A, -1, P) % P, M.G1_B * pow(M.G1_Z * M.G1_A, -1, P) % P]
    f2 = B.f2_mul
    g2_c = [M.G2_A, M.G2_B, M.G2_Z, B.f2_neg(f2(M.G2_B, B.f2_inv(M.G2_A))), f2(M.G2_B, B.f2_inv(f2(M.G2_Z, M.G2_A))), M.PSI_CX, M.PSI_CY]
    return {"kG1Consts": g1_c, "kG1Iso": [c for t in M.G1_TABLES for c in t],
            "kG2Consts": g2_c, "kG2Iso": [c for t in M.G2_TABLES for c in t]}


def table_limbs(values):
    out = []
    for v in values:
        for c in (v if isinstance(v, tuple) else (v,)):
            out += limbs(c)
    return out


def c_source():
    lines = []
    for name, vals in tables().items():
        g2 = isinstance(vals[0], tuple)
        lines.append(f"__constant__ uint32_t {name}[{len(vals)}]{'[2]' if g2 else ''}[12] = {{")
        for v in vals:
            rows = [", ".join(f"0x{w:08x}u" for w in limbs(c)) for c in (v if g2 else (v,))]
            lines.append("    {" + ("{" + "}, {".join(rows) + "}" if g2 else rows[0]) + "},")
        lines.append("};")
    return "\n".join(lines)


def main():
    check_g1_point_count()
    check_g1_iso_on_curve()
    check_g1_iso_additive()
    assert find_z_sswu_g1() == M.G1_Z
    check_g2_against_vector()
    print(c_source())


if __name__ == "__main__":
    main()
