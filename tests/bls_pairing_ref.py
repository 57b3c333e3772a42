"""BLS12-381 pairing reference -- TEST INFRASTRUCTURE ONLY (the library's pairing is ethrex_b200/csrc/bls_pairing.cu).

An independent statement of the pairing, deliberately unlike the device code: Fp12 is the degree-12 field
Fp[w]/(w^12 - 2 w^6 + 2) (no tower), G2 points are untwisted into E(Fp12): y^2 = x^3 + 4, the Miller loop uses affine
chord-and-tangent lines over |x| = 0xd201000000010000, and the final exponentiation is the generic power (p^12 - 1)/r.
Without the conjugation for negative x this is a different (but equally non-degenerate, bilinear) pairing from the
optimal ate one the device computes, so only "is the product one" and bilinearity compare across the two.

Also: Fp2 = Fp[u]/(u^2 + 1) arithmetic and its square root, G2 (the twist y^2 = x^3 + 4(1 + u)) in affine coordinates,
the 96-byte compressed ZCash form of G2 points, and the EIP-2537 128 / 256-byte encodings of G1 / G2."""
import bls_ref as bls

P, R = bls.P, bls.R
X_ABS = 0xD201000000010000  # |x|, x = -0xd201000000010000
G1 = bls.G1
G2 = ((0x024AA2B2F08F0A91260805272DC51051C6E47AD4FA403B02B4510B647AE3D1770BAC0326A805BBEFD48056C8C121BDB8,
       0x13E02B6052719F607DACD3A088274F65596BD0D09920B61AB5DA61BBDC7F5049334CF11213945D57E5AC7D055D042B7E),
      (0x0CE5D527727D6E118CC9CDC6DA2E351AADFD9BAA8CBDD3A76D429A695160D12C923AC9CC3BACA289E193548608B82801,
       0x0606C4A02EA734CC32ACD2B02BC28B99CB3E287E85A763AF267492AB572E99AB3F370D275CEC1DA1AAA9075FF05F79BE))
# the compressed generator of G2, a published constant (the first point of every BLS12-381 G2 test suite)
G2_COMPRESSED = bytes.fromhex("93e02b6052719f607dacd3a088274f65596bd0d09920b61ab5da61bbdc7f5049334cf11213945d57e5ac7d055d042b7e"
                              "024aa2b2f08f0a91260805272dc51051c6e47ad4fa403b02b4510b647ae3d1770bac0326a805bbefd48056c8c121bdb8")
B2 = (4, 4)  # 4 (1 + u)


# ---- Fp2 = Fp[u]/(u^2 + 1): pairs (c0, c1)
def f2_add(a, b): return ((a[0] + b[0]) % P, (a[1] + b[1]) % P)
def f2_sub(a, b): return ((a[0] - b[0]) % P, (a[1] - b[1]) % P)
def f2_neg(a): return (-a[0] % P, -a[1] % P)
def f2_mul(a, b): return ((a[0] * b[0] - a[1] * b[1]) % P, (a[0] * b[1] + a[1] * b[0]) % P)
def f2_sqr(a): return f2_mul(a, a)


def f2_inv(a):
    d = pow((a[0] * a[0] + a[1] * a[1]) % P, -1, P)
    return (a[0] * d % P, -a[1] * d % P)


def f2_pow(a, e):
    acc = (1, 0)
    while e:
        if e & 1:
            acc = f2_mul(acc, a)
        a = f2_sqr(a)
        e >>= 1
    return acc


def f2_sqrt(a):
    """a square root of a in Fp2, or None: through the norm a0^2 + a1^2 and square roots in Fp (p = 3 mod 4)"""
    if a == (0, 0):
        return (0, 0)
    n = (a[0] * a[0] + a[1] * a[1]) % P
    s = pow(n, (P + 1) // 4, P)
    if s * s % P != n:
        return None
    half = pow(2, -1, P)
    for t in ((a[0] + s) * half % P, (a[0] - s) * half % P):
        x0 = pow(t, (P + 1) // 4, P)
        if x0 * x0 % P == t and x0:
            x = (x0, a[1] * pow(2 * x0, -1, P) % P)
            if f2_sqr(x) == a:
                return x
    # a = c0 with c0 a non-square in Fp: sqrt = sqrt(-c0) u
    y = pow(-a[0] % P, (P + 1) // 4, P)
    return (0, y) if a[1] == 0 and y * y % P == -a[0] % P else None


# ---- G2 on the twist, affine, None = identity
def g2_on_curve(q):
    if q is None:
        return True
    x, y = q
    return f2_sqr(y) == f2_add(f2_mul(f2_sqr(x), x), B2)


def g2_add(p, q):
    if p is None:
        return q
    if q is None:
        return p
    (x1, y1), (x2, y2) = p, q
    if x1 == x2:
        if f2_add(y1, y2) == (0, 0):
            return None
        xx = f2_sqr(x1)
        lam = f2_mul(f2_add(f2_add(xx, xx), xx), f2_inv(f2_add(y1, y1)))
    else:
        lam = f2_mul(f2_sub(y2, y1), f2_inv(f2_sub(x2, x1)))
    x3 = f2_sub(f2_sub(f2_sqr(lam), x1), x2)
    return x3, f2_sub(f2_mul(lam, f2_sub(x1, x3)), y1)


def g2_neg(q):
    return None if q is None else (q[0], f2_neg(q[1]))


def g2_mul(k, q, reduce=True):
    if reduce:
        k %= R
    acc = None
    while k:
        if k & 1:
            acc = g2_add(acc, q)
        q = g2_add(q, q)
        k >>= 1
    return acc


def g2_in_subgroup(q):
    return g2_mul(R, q, reduce=False) is None


def g1_in_subgroup(p):
    acc, k, q = None, R, p
    while k:
        if k & 1:
            acc = bls.add(acc, q)
        q = bls.add(q, q)
        k >>= 1
    return acc is None


def _larger(y):
    """the ZCash sign bit of y in Fp2: y.c1 > (p-1)/2, or y.c1 = 0 and y.c0 > (p-1)/2"""
    h = (P - 1) // 2
    return y[1] > h or (y[1] == 0 and y[0] > h)


def g2_compress(q) -> bytes:
    if q is None:
        return bytes([0xC0]) + bytes(95)
    (x0, x1), y = q
    b = bytearray(x1.to_bytes(48, "big") + x0.to_bytes(48, "big"))
    b[0] |= 0x80 | (0x20 if _larger(y) else 0)
    return bytes(b)


def g2_decompress(b: bytes):
    """-> point, None (identity); raises ValueError on anything c-kzg / blst would refuse"""
    if len(b) != 96 or not b[0] & 0x80:
        raise ValueError("not a compressed point")
    x1 = int.from_bytes(b[:48], "big") & ((1 << 381) - 1)
    x0 = int.from_bytes(b[48:], "big")
    if b[0] & 0x40:
        if b[0] & 0x20 or x1 or x0:
            raise ValueError("malformed infinity")
        return None
    if x0 >= P or x1 >= P:
        raise ValueError("coordinate >= p")
    x = (x0, x1)
    y = f2_sqrt(f2_add(f2_mul(f2_sqr(x), x), B2))
    if y is None:
        raise ValueError("not on the curve")
    if _larger(y) != bool(b[0] & 0x20):
        y = f2_neg(y)
    return x, y


def g2_random_point(seed: int):
    """an on-curve point of the twist from a deterministic x (almost surely outside the order-r subgroup)"""
    x0 = seed
    while True:
        x = (x0 % P, (7 * x0 + 3) % P)
        y = f2_sqrt(f2_add(f2_mul(f2_sqr(x), x), B2))
        if y is not None:
            return x, y
        x0 += 1


def g1_random_point(seed: int):
    x = seed % P
    while True:
        rhs = (x ** 3 + 4) % P
        y = pow(rhs, (P + 1) // 4, P)
        if y * y % P == rhs:
            return x, y
        x += 1


# ---- EIP-2537 encodings: each Fp is 16 zero bytes then 48 bytes big-endian; all-zero = identity
def fp64(v: int) -> bytes:
    return bytes(16) + v.to_bytes(48, "big")


def g1_eip2537(p) -> bytes:
    return bytes(128) if p is None else fp64(p[0]) + fp64(p[1])


def g2_eip2537(q) -> bytes:
    return bytes(256) if q is None else fp64(q[0][0]) + fp64(q[0][1]) + fp64(q[1][0]) + fp64(q[1][1])


def g1_from_eip2537(b: bytes):
    x, y = int.from_bytes(b[16:64], "big"), int.from_bytes(b[80:128], "big")
    return None if x == y == 0 else (x, y)


def g2_from_eip2537(b: bytes):
    v = [int.from_bytes(b[64 * i + 16:64 * i + 64], "big") for i in range(4)]
    return None if not any(v) else ((v[0], v[1]), (v[2], v[3]))


# ---- Fp12 = Fp[w]/(w^12 - 2 w^6 + 2): lists of 12 coefficients
def f12_mul(a, b):
    t = [0] * 23
    for i, ai in enumerate(a):
        if ai:
            for j, bj in enumerate(b):
                t[i + j] += ai * bj
    for k in range(22, 11, -1):  # w^k = 2 w^(k-6) - 2 w^(k-12)
        c = t[k]
        if c:
            t[k - 6] += 2 * c
            t[k - 12] -= 2 * c
    return [c % P for c in t[:12]]


def f12_one():
    return [1] + [0] * 11


def f12_pow(a, e):
    acc = f12_one()
    for bit in bin(e)[2:]:
        acc = f12_mul(acc, acc)
        if bit == "1":
            acc = f12_mul(acc, a)
    return acc


def _embed2(a):
    """a0 + a1 u -> Fp12 with u = w^6 - 1 (w^6 satisfies W^2 - 2W + 2 = 0, so (W - 1)^2 = -1)"""
    out = [0] * 12
    out[0], out[6] = (a[0] - a[1]) % P, a[1] % P
    return out


_W = [0, 1] + [0] * 10
_W_INV = f12_pow(_W, P ** 12 - 2)  # one-off: untwisting divides by w^2 and w^3
_W_INV2, _W_INV3 = f12_mul(_W_INV, _W_INV), f12_mul(f12_mul(_W_INV, _W_INV), _W_INV)


def untwist(q):
    """(x', y') on y^2 = x^3 + 4(1+u) -> (x' / w^2, y' / w^3) on y^2 = x^3 + 4 over Fp12"""
    return f12_mul(_embed2(q[0]), _W_INV2), f12_mul(_embed2(q[1]), _W_INV3)


def miller_loop(p, q):
    """f_{|x|,Q}(P) with affine lines in Fp12 (P in G1, Q in G2, neither the identity)"""
    if p is None or q is None:
        return f12_one()
    px, py = [p[0] % P] + [0] * 11, [p[1] % P] + [0] * 11
    f, t = f12_one(), q
    for bit in bin(X_ABS)[3:]:
        f = f12_mul(f12_mul(f, f), _line(t, t, px, py))
        t = g2_add(t, t)
        if bit == "1":
            f = f12_mul(f, _line(t, q, px, py))
            t = g2_add(t, q)
    return f


def _line(t, q, px, py):
    """the line through untwist(t) and untwist(q) (tangent when equal), evaluated at (px, py)"""
    (x1, y1), (x2, y2) = t, q
    if t == q:
        xx = f2_sqr(x1)
        lam = f2_mul(f2_add(f2_add(xx, xx), xx), f2_inv(f2_add(y1, y1)))
    else:
        lam = f2_mul(f2_sub(y2, y1), f2_inv(f2_sub(x2, x1)))
    # untwisted slope: (lam w^-3 dy) / (w^-2 dx) = lam / w
    X1, Y1 = untwist(t)
    lam12 = f12_mul(_embed2(lam), _W_INV)
    dx = [(a - b) % P for a, b in zip(px, X1)]
    return [(a - b - c) % P for a, b, c in zip(py, Y1, f12_mul(lam12, dx))]


FINAL_EXP = (P ** 12 - 1) // R


def pairing(p, q):
    return f12_pow(miller_loop(p, q), FINAL_EXP)


def pairing_check(pairs) -> bool:
    """prod e(P_i, Q_i) == 1, one final exponentiation for the product"""
    f = f12_one()
    for p, q in pairs:
        f = f12_mul(f, miller_loop(p, q))
    return f12_pow(f, FINAL_EXP) == f12_one()
