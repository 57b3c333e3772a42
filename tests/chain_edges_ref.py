"""Edges of the device's scalar-multiplication chains -- TEST INFRASTRUCTURE ONLY.

Every precompile composes the complete XYZZ additions of csrc/curve.cuh (xyzz_add, xyzz_add_mixed) into a chain: a
double-and-add over a raw 256-bit scalar (xyzz_scalar_mul), the ECDSA ladder (secp_lincomb), the cofactor-clearing chains of
map-to-curve (mul_u64 and the psi chain of bls_map.cu) and the point-evaluation combine (kzg_verify_combine).  An addition
inside such a chain meets a doubling (acc = q), a cancellation (acc = -q) or an identity operand with probability about
2^-250 on random input, but every input below is calldata, so a caller reaches those branches on purpose.

Tracers replay one device chain in the device's order of operations (MSB first, which is not the oracles' order) over a
group given as an object with zero / add / neg / mul: `Logs(n)`, the discrete logs of a cyclic group of order n, or
`Points(add, neg)`, an affine group law.  At every addition they record (step, kind) unless the kind is generic.
Constructors build precompile inputs whose chain meets a chosen kind at a chosen step; each returns `Case`s."""
import random
from typing import NamedTuple

import bls12_map_ref as M
import bls_pairing_ref as B
import bls_ref as bls
import pairing_stages_ref as S
import pyref
import secp256k1_ref as k1
import secp256r1_ref as r1

GENERIC, DOUBLE, CANCEL, IDENTITY, INFINITY = "generic", "double", "cancel", "identity", "infinity"


class Case(NamedTuple):
    data: bytes   # the precompile input
    event: str    # DOUBLE, CANCEL or IDENTITY at `step`; INFINITY: the map's output is the identity
    step: tuple   # (addition, bit index) of the tracer's record, or ("output", 0)
    label: str
    params: dict  # what the constructor chose (discrete logs included), for the tracers


# ---- groups -------------------------------------------------------------------------------------------------------------------
class Logs:
    """Z/n: the discrete logs of a cyclic group of order n, 0 the identity"""
    zero = 0

    def __init__(self, n):
        self.n = n

    def add(self, a, b):
        return (a + b) % self.n

    def neg(self, a):
        return -a % self.n

    def mul(self, k, a):
        return k * a % self.n


class Points:
    """an affine group law, None the identity"""
    zero = None

    def __init__(self, add, neg):
        self.add, self.neg = add, neg

    def mul(self, k, p):
        acc = None
        while k:
            if k & 1:
                acc = self.add(acc, p)
            p = self.add(p, p)
            k >>= 1
        return acc


def kind(g, acc, q):
    """what a complete addition acc + q meets: the order of the checks is xyzz_add's"""
    if q == g.zero or acc == g.zero:
        return IDENTITY
    if acc == q:
        return DOUBLE
    if acc == g.neg(q):
        return CANCEL
    return GENERIC


class Trace:
    def __init__(self, g):
        self.g, self.events = g, []

    def add(self, acc, q, step):
        k = kind(self.g, acc, q)
        if k != GENERIC:
            self.events.append((step, k))
        return self.g.add(acc, q)

    def exceptional(self):
        return [(s, k) for s, k in self.events if k in (DOUBLE, CANCEL)]


def _neg_xy(p, mod):
    return None if p is None else (p[0], -p[1] % mod)


BN_G1 = Points(pyref.g1_add, lambda p: _neg_xy(p, pyref.P))
BLS_G1 = Points(bls.add, lambda p: _neg_xy(p, bls.P))
BLS_G2 = Points(B.g2_add, B.g2_neg)
K1 = Points(k1.add, lambda p: _neg_xy(p, k1.P))
R1 = Points(r1.add, r1.neg)


# ---- tracers --------------------------------------------------------------------------------------------------------------------
def scalar_mul(tr, k, p, tag="add"):
    """xyzz_scalar_mul: 256 steps, each a doubling, then a mixed add of p when bit i of k is set"""
    acc = tr.g.zero
    for i in range(255, -1, -1):
        acc = tr.g.add(acc, acc)
        if k >> i & 1:
            acc = tr.add(acc, p, (tag, i))
    return acc


def wnaf(k):
    """secp_wnaf: 257 width-5 NAF digits of k < 2^256, least significant first"""
    out = []
    for _ in range(257):
        d = 0
        if k & 1:
            d = k & 31
            if d >= 16:
                d -= 32
            k -= d
        out.append(d)
        k >>= 1
    assert k == 0
    return out


def lincomb(tr, u1, u2, r, gen):
    """secp_lincomb: u1 gen + u2 r; per step i = 256 .. 0 a doubling, the R-term add at a nonzero wNAF digit of u2, then the
    G-window add of gtab[w - 1] = w gen when i % 12 == 0 and the 12-bit window w of u1 at i is nonzero"""
    g = tr.g
    r2 = g.add(r, r)
    rt = [r]
    for _ in range(7):
        rt.append(g.add(rt[-1], r2))
    naf = wnaf(u2)
    acc = g.zero
    for i in range(256, -1, -1):
        acc = g.add(acc, acc)
        d = naf[i]
        if d:
            q = rt[abs(d) >> 1]
            acc = tr.add(acc, g.neg(q) if d < 0 else q, ("R", i))
        if i % 12 == 0 and i < 256:
            w = u1 >> i & 4095
            if w:
                acc = tr.add(acc, g.mul(w, gen), ("G", i))
    return acc


def mul_u64(tr, k, p, tag="mul"):
    """bls_map.cu's mul_u64: acc = p, then MSB first from bit 62 - clz(k): a doubling, then xyzz_add of p at a set bit"""
    acc = p
    for i in range(k.bit_length() - 2, -1, -1):
        acc = tr.g.add(acc, acc)
        if k >> i & 1:
            acc = tr.add(acc, p, (tag, i))
    return acc


def clear_cofactor_g2(tr, p):
    """bls_map.cu's G2 clear_cofactor (RFC 9380 G.3) in the device's order, over real points of the twist"""
    g = tr.g

    def mul_z(q, tag):
        return g.neg(mul_u64(tr, M.Z_ABS, q, tag))
    t1 = mul_z(p, "z1")
    t2 = M.psi(p)
    t3 = M.psi(M.psi(g.add(p, p)))
    t3 = tr.add(t3, g.neg(t2), ("psi", 0))
    t2 = tr.add(t2, t1, ("psi", 1))
    t3 = tr.add(t3, mul_z(t2, "z2"), ("psi", 2))
    t3 = tr.add(t3, g.neg(t1), ("psi", 3))
    return tr.add(t3, g.neg(p), ("psi", 4))


def map_g1(tr, u):
    """MAP_FP_TO_G1 as the device runs it: sswu, iso_map (its vanishing denominator recorded), h_eff by mul_u64"""
    pt = M.iso_map(M.Fp, M.G1_TABLES, M.sswu(M.Fp, M.G1_A, M.G1_B, M.G1_Z, u))
    if pt is None:
        tr.events.append((("iso_map", 0), IDENTITY))
    return mul_u64(tr, M.H_EFF_G1, pt, "heff")


def map_g2(tr, u):
    pt = M.iso_map(M.Fp2, M.G2_TABLES, M.sswu(M.Fp2, M.G2_A, M.G2_B, M.G2_Z, u))
    if pt is None:
        tr.events.append((("iso_map", 0), IDENTITY))
    return clear_cofactor_g2(tr, pt)


def kzg_combine(tr, c, z, y, pi, gen):
    """kzg_verify_combine: [z] pi by xyzz_scalar_mul, + C (mixed), + (-[y] gen)"""
    g = tr.g
    acc = scalar_mul(tr, z, pi, "z")
    acc = tr.add(acc, c, ("C", 0))
    yg = scalar_mul(tr, y, gen, "y")
    return tr.add(acc, g.neg(yg), ("-yG", 0))


def run(tracer, g, *args):
    """(final value, trace) of one tracer over group g"""
    tr = Trace(g)
    return tracer(tr, *args), tr


# ---- raw-scalar chains: ecMul (BN254 G1) and the EIP-2537 MSM terms (BLS12-381 G1 / G2) ---------------------------------------
# At the add of bit i the prefix is A = k >> i (odd), acc = (A - 1) P and q = P.  With P of prime order r the add doubles when
# A = 2 (mod r) and cancels when A = 0 (mod r); A < 2^256 and A odd leave A = m r or m r + 2 with m odd, and the add sits at
# bit s when k = A 2^s + low, low < 2^s.
def exceptional_prefixes(r):
    """{A: kind} over every odd A < 2^256 with A = 0 or 2 (mod r): all multiples of r below 2^256, both offsets"""
    out = {}
    for q in range((1 << 256) // r + 1):
        for off, kd in ((0, CANCEL), (2, DOUBLE)):
            a = q * r + off
            if a & 1 and a < 1 << 256:
                out[a] = kd
    return out


def raw_scalar_edges(r, seed):
    """[(k, kind, bit, (m, s))]: every exceptional prefix A = m r (+ 2) at every shift s with A 2^s < 2^256, and
    low in {0, 1, 2^s - 1} plus one random value below 2^s"""
    rng = random.Random(seed)
    out = []
    for a, kd in sorted(exceptional_prefixes(r).items()):
        s = 0
        while a << s < 1 << 256:
            for low in sorted({0, min(1, (1 << s) - 1), (1 << s) - 1, rng.randrange(1 << s)}):
                out.append((a << s | low, kd, s, (a // r, s)))
            s += 1
    return out


def _cube_roots_of_unity(q):
    w = next(w for w in (pow(g, (q - 1) // 3, q) for g in range(2, 64)) if w != 1)
    return sorted({w, w * w % q})


def endomorphism_eigenvalues():
    """{curve: [lambda]}: the eigenvalues on the prime-order group of phi(x, y) = (beta x, y) on BN254 G1 and BLS12-381 G1
    (both cube roots of unity mod r, each checked against some cube root beta on the generator) and of psi on BLS12-381 G2
    (the p-power Frobenius of the twist, so [p mod r]; checked on the generator)"""
    out = {}
    for name, r, p, gen, mul in (("bn254_g1", pyref.R, pyref.P, pyref.G1_GEN, pyref.g1_mul), ("bls12_381_g1", bls.R, bls.P, bls.G1, bls.mul)):
        betas = _cube_roots_of_unity(p)
        lams = _cube_roots_of_unity(r)
        for lam in lams:
            x, y = mul(lam, gen)
            assert y == gen[1] and any(x == b * gen[0] % p for b in betas), name
        out[name] = lams
    lam = B.P % B.R
    assert M.psi(B.G2) == B.g2_mul(lam, B.G2)
    out["bls12_381_g2"] = [lam]
    return out


def scalar_cases(curve, seed=0x7):
    """[(k, event, step, label)] for one curve: the raw-scalar edges, then lambda - 1, lambda, lambda + 1"""
    r = pyref.R if curve == "bn254_g1" else bls.R
    out = [(k, kd, ("add", s), f"{m}r{'+2' if kd == DOUBLE else ''}<<{s}|{k & ((1 << s) - 1):#x}") for k, kd, s, (m, _) in raw_scalar_edges(r, seed)]
    for lam in endomorphism_eigenvalues()[curve]:
        out += [(lam + d, GENERIC, None, f"lambda{d:+d}") for d in (-1, 0, 1)]
    return out


# ---- the ECDSA ladder ---------------------------------------------------------------------------------------------------------
def _before(u1, u2, op, i):
    """(a, b): just before the op ("R" or "G") addition at step i the accumulator is a G + b R"""
    naf = wnaf(u2)
    b = sum(d << (k - i) for k, d in enumerate(naf) if k > i or (op == "G" and k == i))
    a = sum((u1 >> j & 4095) << (j - i) for j in range(0, 256, 12) if j > i)
    return a, b


def solve_t(u1, u2, op, i, kd, n):
    """the discrete log t of R for which the op addition at step i meets kd (DOUBLE or CANCEL)"""
    a, b = _before(u1, u2, op, i)
    sign = 1 if kd == DOUBLE else -1
    if op == "R":  # a + b t = +-d t
        t = a * pow(sign * wnaf(u2)[i] - b, -1, n) % n
    else:  # a + b t = +-w
        t = (sign * (u1 >> i & 4095) - a) * pow(b, -1, n) % n
    assert t
    return t


def ladder_params(n, seed=0xEC):
    """[(u1, u2, op, i, kind, label)]: the G-window add at the top window (252, four bits left), a middle one and 0, with
    low = 0 (a cancellation leaves Q = O) and random low (the ladder passes through O and continues); the R-term add at steps
    251, 130 and 0 below a lone G window; the R-term add at a -1 wNAF digit"""
    rng = random.Random(seed)
    out = []
    for i, w in ((252, 0x9), (132, 0xA5C), (0, 0x3C1)):
        for low in sorted({0, rng.randrange(1 << i)}):
            for kd in (DOUBLE, CANCEL):
                out.append((w << i | low, 1 << i, "G", i, kd, f"G@{i} low={'0' if low == 0 else 'rand'}"))
    for i, m, w in ((251, 252, 0xB), (130, 144, 0x7E5), (0, 12, 0x123)):
        low = rng.randrange(1 << (i - 6)) if i > 6 else 0
        for kd in (DOUBLE, CANCEL):
            out.append((w << m, (1 << i) + low, "R", i, kd, f"R@{i}"))
    for kd in (DOUBLE, CANCEL):  # 31 2^100 = 2^105 - 2^100: digits -1 at 100 and +1 at 105
        out.append((0x5A5 << 120, 31 << 100 | rng.randrange(1 << 90), "R", 100, kd, "R@100 digit=-1"))
    cases = []
    for u1, u2, op, i, kd, label in out:
        assert 0 < u1 < n and 0 < u2 < n
        cases.append(dict(u1=u1, u2=u2, t=solve_t(u1, u2, op, i, kd, n), op=op, i=i, kind=kd, label=label))
    return cases


def ecrecover_input(u1, u2, t):
    """sig | msg (65 + 32 bytes) whose recovery runs secp_lincomb(u1, u2, R = tG): r = x(R), recid = y(R)'s parity,
    s = u2 r, z = -u1 r (mod n), so the device's u1 = -z / r and u2 = s / r are the chosen ones"""
    R = k1.mul(t, k1.G)
    assert R[0] < k1.N
    r, n = R[0], k1.N
    s, z = u2 * r % n, -u1 * r % n
    return r.to_bytes(32, "big") + s.to_bytes(32, "big") + bytes([R[1] & 1]) + z.to_bytes(32, "big")


def p256_input(u1, u2, t):
    """P256VERIFY input under Q = tG with the device's u1 = h / s, u2 = r / s: forged when R' = u1 G + u2 Q is a point,
    else any r (the item cannot verify)"""
    q = r1.mul(t, r1.G)
    if (u1 + u2 * t) % r1.N:
        h, r, s = r1.forge(q, u1, u2)
    else:
        r = 0x1234567
        s = r * pow(u2, -1, r1.N) % r1.N
        h = u1 * s % r1.N
    return r1.encode(h, r, s, q)


def ecrecover_cases():
    return [Case(ecrecover_input(p["u1"], p["u2"], p["t"]), p["kind"], (p["op"], p["i"]), p["label"], p) for p in ladder_params(k1.N)]


def p256_cases():
    return [Case(p256_input(p["u1"], p["u2"], p["t"]), p["kind"], (p["op"], p["i"]), p["label"], p) for p in ladder_params(r1.N)]


def ecrecover_ladder(sig, msg):
    """(u1, u2, R) as secp_recover derives them, or None where it stops before the ladder"""
    r, s, recid = int.from_bytes(sig[:32], "big"), int.from_bytes(sig[32:64], "big"), sig[64]
    if not (0 < r < k1.N and 0 < s < k1.N) or recid > 1:
        return None
    R = k1.lift_x(r, recid & 1)
    z = int.from_bytes(msg, "big") % k1.N
    ri = pow(r, -1, k1.N)
    return -z * ri % k1.N, s * ri % k1.N, R


def p256_ladder(inp):
    h, r, s, qx, qy = r1.decode(inp)
    w = pow(s, -1, r1.N)
    return h % r1.N * w % r1.N, r * w % r1.N, (qx, qy)


# ---- map-to-curve ---------------------------------------------------------------------------------------------------------------
class IsoCurve:
    """E' / E2': y^2 = x^3 + A x + B over Fp / Fp2 (A != 0) in affine coordinates, None the identity"""

    def __init__(self, F, A, Bc, Z, tables, order, primes):
        self.F, self.A, self.B, self.Z, self.tables, self.order, self.primes = F, A, Bc, Z, tables, order, primes

    def div(self, a, b):
        return self.F.mul(a, self.F.inv0(b))

    def rhs(self, x):
        F = self.F
        return F.add(F.mul(F.add(F.mul(x, x), self.A), x), self.B)

    def on_curve(self, p):
        return p is None or self.F.mul(p[1], p[1]) == self.rhs(p[0])

    def neg(self, p):
        return None if p is None else (p[0], self.F.neg(p[1]))

    def add(self, p, q):
        F = self.F
        if p is None:
            return q
        if q is None:
            return p
        (x1, y1), (x2, y2) = p, q
        if x1 == x2:
            if F.add(y1, y2) == F.zero:
                return None
            xx = F.mul(x1, x1)
            lam = self.div(F.add(F.add(F.add(xx, xx), xx), self.A), F.add(y1, y1))
        else:
            lam = self.div(F.sub(y2, y1), F.sub(x2, x1))
        x3 = F.sub(F.sub(F.mul(lam, lam), x1), x2)
        return x3, F.sub(F.mul(lam, F.sub(x1, x3)), y1)

    def mul(self, k, p):
        return Points(self.add, self.neg).mul(k, p)

    def random_point(self, rng):
        while True:
            x = rng.randrange(M.P) if self.F is M.Fp else (rng.randrange(M.P), rng.randrange(M.P))
            y = self.F.sqrt(self.rhs(x))
            if y is not None:
                return x, y

    def sswu(self, u):
        return M.sswu(self.F, self.A, self.B, self.Z, u)

    def _quadratic_roots(self, a, b, c):
        F = self.F
        d = F.sqrt(F.sub(F.mul(b, b), F.mul(F.add(F.add(a, a), F.add(a, a)), c)))
        if d is None:
            return []
        return [self.div(F.add(F.neg(b), e), F.add(a, a)) for e in {d, F.neg(d)}]

    def preimages(self, x):
        """every u with x(sswu(u)) = x, w = Z u^2: the x1 branch solves (x (-A/B) - 1)(w^2 + w) = 1, the Z u^2 x1 branch
        (-B/A)(w^2 + w + 1) = x (w + 1); then u = +-sqrt(w / Z), kept where the forward map agrees"""
        F = self.F
        c1 = F.sub(F.mul(x, F.neg(self.div(self.A, self.B))), F.one)
        ba = F.neg(self.div(self.B, self.A))
        ws = self._quadratic_roots(c1, c1, F.neg(F.one)) + self._quadratic_roots(ba, F.sub(ba, x), F.sub(ba, x))
        out = set()
        for w in ws:
            u = F.sqrt(self.div(w, self.Z))
            if u is not None:
                out |= {u for u in (u, F.neg(u)) if self.sswu(u)[0] == x}
        return sorted(out)


E1 = IsoCurve(M.Fp, M.G1_A, M.G1_B, M.G1_Z, M.G1_TABLES, bls.R * S.BLS_H1, S.BLS_G1.factors)
E2 = IsoCurve(M.Fp2, M.G2_A, M.G2_B, M.G2_Z, M.G2_TABLES, bls.R * S.BLS_H2, S.BLS_G2.factors)


# polynomials over Fp, coefficient lists in ascending powers
def _trim(a):
    while a and a[-1] == 0:
        a.pop()
    return a


def _divmod(a, b):
    a, q = list(a), [0] * max(0, len(a) - len(b) + 1)
    inv = pow(b[-1], -1, M.P)
    while len(_trim(a)) >= len(b):
        c, d = a[-1] * inv % M.P, len(a) - len(b)
        q[d] = c
        for j, bj in enumerate(b):
            a[d + j] = (a[d + j] - c * bj) % M.P
    return _trim(q), a


def _mulmod(a, b, f):
    t = [0] * (len(a) + len(b))
    for i, ai in enumerate(a):
        for j, bj in enumerate(b):
            t[i + j] += ai * bj
    return _divmod([c % M.P for c in t], f)[1]


def _powmod(a, e, f):
    acc = [1]
    for bit in bin(e)[2:]:
        acc = _mulmod(acc, acc, f)
        if bit == "1":
            acc = _mulmod(acc, a, f)
    return acc


def _gcd(a, b):
    a, b = _trim(list(a)), _trim(list(b))
    while b:
        a, b = b, _divmod(a, b)[1]
    inv = pow(a[-1], -1, M.P)
    return [c * inv % M.P for c in a]


def roots_fp(f, seed=11):
    """the distinct roots in Fp of f: gcd(f, x^p - x), then split by gcd((x + a)^((p - 1)/2) - 1, h) (Cantor-Zassenhaus)"""
    rng = random.Random(seed)
    xp = _powmod([0, 1], M.P, f)
    h = _gcd(f, _trim([(c - (1 if i == 1 else 0)) % M.P for i, c in enumerate(xp + [0] * max(0, 2 - len(xp)))]))

    def split(h):
        if len(h) == 1:
            return []
        if len(h) == 2:
            return [-h[0] % M.P]
        while True:
            g = _powmod([rng.randrange(M.P), 1], (M.P - 1) // 2, h)
            g = _gcd(h, _trim([(g[0] - 1) % M.P] + g[1:]) or [0])
            if 1 < len(g) < len(h):
                return split(g) + split(_divmod(h, g)[0])
    return sorted(split(h))


def g1_kernel_inputs():
    """{root x0 of x_den in Fp: [u]}: iso_map's denominator vanishes at x0; the u whose SSWU point has x = x0"""
    roots = roots_fp(list(M.G1_XDEN) + [1])
    for x0 in roots:
        assert M.poly(M.Fp, M.G1_XDEN, x0, monic=True) == 0
    return {x0: (E1.preimages(x0) if M.Fp.sqrt(E1.rhs(x0)) is not None else []) for x0 in roots}


def g2_kernel_root():
    """(x0, g(x0)): x_den = x^2 + c1 x + c0 over Fp2 has discriminant 0, so its only root is x0 = -c1/2"""
    c0, c1 = M.G2_XDEN
    F = M.Fp2
    assert F.sub(F.mul(c1, c1), F.mul((4, 0), c0)) == F.zero
    x0 = E2.div(F.neg(c1), (2, 0))
    assert M.poly(F, M.G2_XDEN, x0, monic=True) == F.zero
    return x0, E2.rhs(x0)


def torsion_inputs(curve, seed=0x11, tries=24):
    """{(l, k): (point, [u])} for each prime l of the cofactor and each order l^k met: T = (r h / l^e) P for random points P
    of E', its multiples l^j T of every smaller l-power order, and for each order the SSWU preimages of Q, 2Q, 3Q, .. (Q of
    that order) until one has some.  An order whose points have no preimage maps to (None, [])."""
    rng = random.Random(seed)
    out = {}
    for ell, e in sorted(curve.primes.items()):
        for _ in range(4):
            t = curve.mul(curve.order // ell ** e, curve.random_point(rng))
            chain = []
            while t is not None:
                chain.append(t)
                t = curve.mul(ell, t)
            for k, q0 in enumerate(reversed(chain), 1):  # q0 has order l^k
                if out.get((ell, k), (None, []))[1]:
                    continue
                out[(ell, k)] = (None, [])
                for j in range(1, min(tries, ell)):
                    q = curve.mul(j, q0)
                    us = curve.preimages(q[0])
                    if us:
                        out[(ell, k)] = (q, us)
                        break
    return out


def map_cases():
    """(G1 cases, G2 cases, {(l, k): count} per group): every G1 u whose SSWU point is an iso_map kernel point, and the
    preimages of one point of each l-power order l^k met, per prime l of each cofactor.  Each output is the identity."""
    g1, g2 = [], []
    for x0, us in g1_kernel_inputs().items():
        g1 += [Case(M.fp64(u), INFINITY, ("iso_map", 0), f"x_den root {x0:#x}"[:24], dict(u=u, ell=None)) for u in us]
    counts = ({}, {})
    for out, curve, enc, cnt in ((g1, E1, M.fp64, counts[0]), (g2, E2, M.fp2_64, counts[1])):
        for (ell, k), (_, us) in sorted(torsion_inputs(curve).items()):
            cnt[(ell, k)] = len(us)
            out += [Case(enc(u), INFINITY, ("output", 0), f"T_{ell}^{k}", dict(u=u, ell=ell, k=k)) for u in us]
    return g1, g2, counts


# ---- point evaluation: kzg_verify_combine over the known-tau setup of tests/test_gpu_kzg_verify.py ---------------------------
TAU = 0x2F1B7C93D4A5E6F708192A3B4C5D6E7F8091A2B3C4D5E6F708192A3B4C5D6E7F % bls.R
G2_SETUP = B.G2_COMPRESSED + B.g2_compress(B.g2_mul(TAU, B.G2))


def kzg_params(seed=0x4844):
    """[dict(a, c, z, y, kind, step, valid, label)] with pi = [a] G, C = [c] G.  The C add doubles when c = z a and cancels when
    c = -z a; the -[y] G add doubles when z a + c = -y and cancels when z a + c = y.  The item verifies when
    c - y + z a = a tau; each event once valid and once not, where the cancelling -[y] G add's valid item is pi = O, C = [y] G"""
    rng = random.Random(seed)
    R, half = bls.R, pow(2, -1, bls.R)
    out = []

    def item(label, kd, step, a, c, z, y):
        out.append(dict(a=a % R, c=c % R, z=z % R, y=y % R, kind=kd, step=step, valid=(c - y + z * a - a * TAU) % R == 0, label=label))
    for valid in (True, False):
        a, z = rng.randrange(1, R), rng.randrange(1, R)
        extra = 0 if valid else rng.randrange(1, R)
        item(f"C doubles, valid={valid}", DOUBLE, ("C", 0), a, z * a, z, 2 * z * a - a * TAU + extra)
        item(f"C cancels, valid={valid}", CANCEL, ("C", 0), a, -z * a, z, -a * TAU + extra)
        y = -a * TAU * half if valid else rng.randrange(1, R)
        item(f"-yG doubles, valid={valid}", DOUBLE, ("-yG", 0), a, -y - z * a, z, y)
        if valid:
            y = rng.randrange(1, R)
            item("-yG cancels, pi = O, C = [y]G", CANCEL, ("-yG", 0), 0, y, z, y)
        else:
            y = rng.randrange(1, R)
            item("-yG cancels, valid=False", CANCEL, ("-yG", 0), a, y - z * a, z, y)
    return out


def kzg_input(p):
    c, pi = bls.generator_multiples([p["c"], p["a"]])
    return bls.compress(c) + p["z"].to_bytes(32, "big") + p["y"].to_bytes(32, "big") + bls.compress(pi)


def kzg_cases():
    return [Case(kzg_input(p), p["kind"], p["step"], p["label"], p) for p in kzg_params()]
