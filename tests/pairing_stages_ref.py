"""The stages of both device pairings, restated in Python -- TEST INFRASTRUCTURE ONLY.

Shared by tests/test_pairing_stages_host.py (the restatement against independent anchors) and
tests/test_gpu_pairing_conformance.py (the device stages of tests/csrc/pairing_conformance.cu against the restatement).

BLS12-381 (ethrex_b200/csrc/bls_pairing.cuh).  An Fp12 element is the tower value of field_conformance_ref.BLS_FP12:
((a0, a1, a2), (b0, b1, b2)) = sum a_j v^j + sum b_j v^j w over Fp2 pairs, v = w^2, w^6 = xi = 1 + u.  Products and
powers go through the 12 flat Fp coefficients of bls_pairing_ref (Fp[w]/(w^12 - 2 w^6 + 2), the same w, u = w^6 - 1),
converted explicitly by to_flat / from_flat.  The restatement follows the device step by step where the value depends on
the steps -- the projective line coefficients of Costello-Lange-Naehrig 2010 and the mul_014 slot layout
l = c0 + (c1 xP) v + (c2 yP) v w -- and is plain field arithmetic where it does not (f^x, the final exponentiation).

BN254 (ethrex_b200/csrc/bn_pairing.cuh): oracle/pyref_tower.py is already the device algorithm in Python, over the same
tower and with the same tuple layout; this module adds the cofactor data and the anchors.

Cofactor-component points: for each prime l of a cofactor h, a point of order exactly l, a point of the largest order
l^k the group holds, and the sums of those with a subgroup point.  A random curve point has a component of every order
at once, so it cannot show a subgroup check that misses one of them."""
import bls_pairing_ref as B
import bls_ref as bls
import pyref
import pyref_tower as BT

P, R = B.P, B.R
X_ABS = B.X_ABS  # x = -X_ABS
F2_ZERO, F2_ONE = (0, 0), (1, 0)
XI = (1, 1)
TWO_INV = (P + 1) // 2


# ---- Fp12: tower <-> flat -----------------------------------------------------------------------------------------------
def _coeffs(t):
    """the six Fp2 coefficients of w^0 .. w^5"""
    (a0, a1, a2), (b0, b1, b2) = t
    return [a0, b0, a1, b1, a2, b2]


def _tower(cs):
    return ((cs[0], cs[2], cs[4]), (cs[1], cs[3], cs[5]))


def to_flat(t):
    """c0 + c1 u at w^k, u = w^6 - 1: c0 - c1 at w^k, c1 at w^(k + 6)"""
    out = [0] * 12
    for k, (c0, c1) in enumerate(_coeffs(t)):
        out[k] = (c0 - c1) % P
        out[k + 6] = c1 % P
    return out


def from_flat(d):
    return _tower([((d[k] + d[k + 6]) % P, d[k + 6]) for k in range(6)])


ONE = _tower([F2_ONE] + [F2_ZERO] * 5)
ZERO = _tower([F2_ZERO] * 6)
W = _tower([F2_ZERO, F2_ONE] + [F2_ZERO] * 4)


def mul(a, b):
    return from_flat(B.f12_mul(to_flat(a), to_flat(b)))


def sqr(a):
    return mul(a, a)


def power(a, e):
    return from_flat(B.f12_pow(to_flat(a), e))


def conj(a):
    return (a[0], tuple(B.f2_neg(c) for c in a[1]))


def _f2_mul_xi(a):
    return ((a[0] - a[1]) % P, (a[0] + a[1]) % P)


def _f6_mul(a, b):
    c = [F2_ZERO] * 5
    for i in range(3):
        for j in range(3):
            c[i + j] = B.f2_add(c[i + j], B.f2_mul(a[i], b[j]))
    return (B.f2_add(c[0], _f2_mul_xi(c[3])), B.f2_add(c[1], _f2_mul_xi(c[4])), c[2])


def _f6_inv(a):
    A = B.f2_sub(B.f2_sqr(a[0]), _f2_mul_xi(B.f2_mul(a[1], a[2])))
    Bc = B.f2_sub(_f2_mul_xi(B.f2_sqr(a[2])), B.f2_mul(a[0], a[1]))
    C = B.f2_sub(B.f2_sqr(a[1]), B.f2_mul(a[0], a[2]))
    n = B.f2_add(B.f2_mul(a[0], A), _f2_mul_xi(B.f2_add(B.f2_mul(a[2], Bc), B.f2_mul(a[1], C))))
    ni = B.f2_inv(n)
    return (B.f2_mul(A, ni), B.f2_mul(Bc, ni), B.f2_mul(C, ni))


def inv(a):
    """a^-1, and 0 for 0 (the device's convention)"""
    if a == ZERO:
        return ZERO
    # (a0 + a1 w)(a0 - a1 w) = a0^2 - a1^2 v lies in Fp6
    v_a1sq = _f6_mul(a[1], a[1])
    d = tuple(B.f2_sub(x, y) for x, y in zip(_f6_mul(a[0], a[0]), (_f2_mul_xi(v_a1sq[2]), v_a1sq[0], v_a1sq[1])))
    di = _f6_inv(d)
    return (_f6_mul(a[0], di), tuple(B.f2_neg(c) for c in _f6_mul(a[1], di)))


# ---- BLS12-381 stages, as bls_pairing.cuh computes them -------------------------------------------------------------------
FROB1 = [B.f2_pow(XI, k * (P - 1) // 6) for k in range(6)]
FROB2 = [B.f2_pow(XI, k * (P * P - 1) // 6) for k in range(6)]


def frob(a):
    """(sum_k a_k w^k)^p = sum_k conj(a_k) xi^(k (p - 1)/6) w^k"""
    return _tower([B.f2_mul((c[0], -c[1] % P), FROB1[k]) for k, c in enumerate(_coeffs(a))])


def frob2(a):
    return _tower([B.f2_mul(c, FROB2[k]) for k, c in enumerate(_coeffs(a))])


def exp_x(f):
    """conj(f^|x|): f^x wherever conj is the inverse (the cyclotomic subgroup), and this value everywhere else"""
    return conj(power(f, X_ABS))


def final_exponentiate(f0):
    f = mul(conj(f0), inv(f0))
    f = mul(frob2(f), f)
    t = mul(exp_x(f), conj(f))
    t = mul(exp_x(t), conj(t))
    t = mul(exp_x(t), frob(t))
    t = mul(mul(exp_x(exp_x(t)), frob2(t)), conj(t))
    return mul(t, mul(sqr(f), f))


FINAL_EXP_BLS = 3 * (P ** 12 - 1) // R  # the exponent the x-chain computes: the cube of the reduced pairing


def _mul_b2(a):
    return B.f2_mul(a, (4, 4))


def line_double(T):
    """T = (X, Y, Z) homogeneous over Fp2 -> (2T, (c0, c1, c2))"""
    X, Y, Z = T
    s = lambda a: (a[0] * TWO_INV % P, a[1] * TWO_INV % P)  # noqa: E731
    a = s(B.f2_mul(X, Y))
    b, c = B.f2_sqr(Y), B.f2_sqr(Z)
    e = _mul_b2(B.f2_add(B.f2_add(c, c), c))
    f = B.f2_add(B.f2_add(e, e), e)
    g = s(B.f2_add(b, f))
    h = B.f2_sub(B.f2_sqr(B.f2_add(Y, Z)), B.f2_add(b, c))
    i, j, e2 = B.f2_sub(e, b), B.f2_sqr(X), B.f2_sqr(e)
    T2 = (B.f2_mul(a, B.f2_sub(b, f)), B.f2_sub(B.f2_sqr(g), B.f2_add(B.f2_add(e2, e2), e2)), B.f2_mul(b, h))
    return T2, (i, B.f2_add(B.f2_add(j, j), j), B.f2_neg(h))


def line_add(T, q):
    """T homogeneous, q affine over Fp2 -> (T + q, (c0, c1, c2))"""
    X, Y, Z = T
    qx, qy = q
    theta, lam = B.f2_sub(Y, B.f2_mul(qy, Z)), B.f2_sub(X, B.f2_mul(qx, Z))
    c, d = B.f2_sqr(theta), B.f2_sqr(lam)
    e, f, g = B.f2_mul(lam, d), B.f2_mul(Z, c), B.f2_mul(X, d)
    h = B.f2_sub(B.f2_add(e, f), B.f2_add(g, g))
    T2 = (B.f2_mul(lam, h), B.f2_sub(B.f2_mul(theta, B.f2_sub(g, h)), B.f2_mul(e, Y)), B.f2_mul(Z, e))
    return T2, (B.f2_sub(B.f2_mul(theta, qx), B.f2_mul(lam, qy)), B.f2_neg(theta), lam)


def g2_prepare(q):
    """-> (the 68 lines, the final T)"""
    T, lines = (q[0], q[1], F2_ONE), []
    for bit in bin(X_ABS)[3:]:
        T, l = line_double(T)
        lines.append(l)
        if bit == "1":
            T, l = line_add(T, q)
            lines.append(l)
    assert len(lines) == 68
    return lines, T


def line_value(l, p):
    """the sparse element c0 + (c1 xP) v + (c2 yP) v w"""
    sc = lambda a, k: (a[0] * k % P, a[1] * k % P)  # noqa: E731
    return ((l[0], sc(l[1], p[0]), F2_ZERO), (F2_ZERO, sc(l[2], p[1]), F2_ZERO))


def miller(lines, p):
    f, k = ONE, 0
    for bit in bin(X_ABS)[3:]:
        f = mul(sqr(f), line_value(lines[k], p))
        k += 1
        if bit == "1":
            f = mul(f, line_value(lines[k], p))
            k += 1
    return conj(f)


def pair(p, q):
    return final_exponentiate(miller(g2_prepare(q)[0], p))


# ---- cofactors --------------------------------------------------------------------------------------------------------------
def is_probable_prime(n):
    if n < 2:
        return False
    for s in (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37):
        if n % s == 0:
            return n == s
    d, k = n - 1, 0
    while d % 2 == 0:
        d, k = d // 2, k + 1
    for a in (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37, 41):
        x = pow(a, d, n)
        if x in (1, n - 1):
            continue
        for _ in range(k - 1):
            x = x * x % n
            if x == n - 1:
                break
        else:
            return False
    return True


def _factor(h, small):
    """{l: e} of h, given every prime factor but the largest"""
    out, rest = {}, h
    for ell in small:
        while rest % ell == 0:
            out[ell] = out.get(ell, 0) + 1
            rest //= ell
    if rest > 1:
        out[rest] = 1
    assert all(is_probable_prime(ell) for ell in out)
    return out


BLS_H1 = 0x396C8C005555E1568C00AAAB0000AAAB
BN_H2 = 2 * pyref.P - pyref.R  # #E'(Fp2) = r (2p - r) for the BN254 twist
_T1 = -X_ABS + 1  # the trace of E(Fp)
_T2 = _T1 * _T1 - 2 * P  # the trace of E(Fp2)


def _bls_h2():
    """the G2 cofactor: of the sextic twists' orders p^2 + 1 -+ (3 f2 +- t2)/2 (3 f2^2 = 4 p^2 - t2^2), the one r divides and
    that the twist's points satisfy"""
    import math
    f2 = math.isqrt((4 * P * P - _T2 * _T2) // 3)
    assert 3 * f2 * f2 == 4 * P * P - _T2 * _T2
    for n in [P * P + 1 - t for t in ((_T2 + 3 * f2) // 2, (_T2 - 3 * f2) // 2, (-_T2 + 3 * f2) // 2, (-_T2 - 3 * f2) // 2)]:
        if n % R == 0 and B.g2_mul(n, B.g2_random_point(5), reduce=False) is None:
            return n // R
    raise AssertionError("no twist order")


BLS_H2 = _bls_h2()


class CurveGroup:
    """an elliptic curve group E(F) = r h points, affine, None the identity"""

    def __init__(self, name, add, neg, on_curve, random_point, gen, r, h, small):
        self.name, self.add, self.neg, self.on_curve, self.random_point, self.gen, self.r, self.h = name, add, neg, on_curve, random_point, gen, r, h
        self.factors = _factor(h, small)

    def mul(self, k, pt):
        """k pt, k not reduced"""
        acc = None
        while k:
            if k & 1:
                acc = self.add(acc, pt)
            pt = self.add(pt, pt)
            k >>= 1
        return acc

    def order_is(self, pt, n):
        return self.mul(n, pt) is None and all(self.mul(n // ell, pt) is not None for ell in _factor(n, list(self.factors)))

    def component(self, ell, seed):
        """-> (a point of order exactly ell, a point of the largest order ell^k found over a few random points)"""
        e = self.factors[ell]
        exact, best, best_k = None, None, 0
        for s in range(seed, seed + 8):
            q = self.mul(self.r * self.h // ell ** e, self.random_point(s))
            k = 0
            while q is not None and self.mul(ell ** (k + 1), q) is not None:
                k += 1
            if q is None:
                continue
            k += 1  # q has order ell^k
            if k > best_k:
                best, best_k = q, k
            if exact is None:
                exact = self.mul(ell ** (k - 1), q)
            if best_k == e:
                break
        assert exact is not None and self.order_is(exact, ell)
        assert self.order_is(best, ell ** best_k)
        return exact, best, best_k

    def cases(self, seed=0x2537):
        """[(name, point, in the subgroup)]: for each prime l of h, T_l, the largest l-power-order point, and each of them plus
        a subgroup point; then subgroup points (the generator, its negation, [r - 1] of it, small multiples)"""
        sub = self.mul(0xC0FFEE, self.gen)
        out = []
        for ell in sorted(self.factors):
            exact, big, k = self.component(ell, seed + ell % 1000)
            out += [(f"T_{ell}", exact, False), (f"G+T_{ell}", self.add(sub, exact), False)]
            if k > 1:
                out += [(f"T_{ell}^{k}", big, False), (f"G+T_{ell}^{k}", self.add(sub, big), False)]
        out += [("G", self.gen, True), ("-G", self.neg(self.gen), True), ("[r-1]G", self.mul(self.r - 1, self.gen), True),
                ("[2]G", self.mul(2, self.gen), True), ("[3]G", self.mul(3, self.gen), True), ("sub", sub, True)]
        for _, pt, _ in out:
            assert self.on_curve(pt)
        return out


def _g1_neg(p):
    return None if p is None else (p[0], -p[1] % P)


BLS_G1 = CurveGroup("bls12_381_g1", bls.add, _g1_neg, bls.on_curve, B.g1_random_point, B.G1, R, BLS_H1,
                    [3, 11, 10177, 859267, 52437899])
BLS_G2 = CurveGroup("bls12_381_g2", B.g2_add, B.g2_neg, B.g2_on_curve, B.g2_random_point, B.G2, R, BLS_H2,
                    [13, 23, 2713, 11953, 262069])


def _bn_g2_random_point(seed):
    x = seed
    while True:
        rhs = pyref.f2_add(pyref.f2_mul(pyref.f2_mul((x, 1), (x, 1)), (x, 1)), pyref.B_G2)
        y = _bn_f2_sqrt(rhs)
        if y is not None:
            return ((x, 1), y)
        x += 1


def _bn_f2_sqrt(a):
    p = pyref.P
    def sq(v):
        r = pow(v, (p + 1) // 4, p)
        return r if r * r % p == v % p else None
    s = sq((a[0] * a[0] + a[1] * a[1]) % p)
    if s is None:
        return None
    for t in ((a[0] + s) * pow(2, -1, p) % p, (a[0] - s) * pow(2, -1, p) % p):
        x0 = sq(t)
        if x0:
            r = (x0, a[1] * pow(2 * x0, -1, p) % p)
            if pyref.f2_mul(r, r) == (a[0] % p, a[1] % p):
                return r
    return None


BN_G2 = CurveGroup("bn254_g2", pyref.g2_add, lambda q: None if q is None else (q[0], pyref.f2_neg(q[1])), pyref.g2_on_curve,
                   _bn_g2_random_point, pyref.G2_GEN, pyref.R, BN_H2, [10069, 5864401, 1875725156269])
