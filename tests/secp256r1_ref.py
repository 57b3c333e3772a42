"""Python oracle for P256VERIFY (EIP-7951) on secp256r1: curve arithmetic over integers in affine coordinates, and
verification with the rules of include/b200zk.h in order (those of the reference's Crypto::secp256r1_verify through the
p256 crate, and of EIP-7951).

verify(inp160) -> bool, inp = h | r | s | qx | qy (32-byte big-endian words).  The constructions below build inputs that
reach the edges of those rules: forged signatures for any key, x(R') >= n, equal points inside an addition, R' = O.
"""
P = 2**256 - 2**224 + 2**192 + 2**96 - 1
N = 0xFFFFFFFF00000000FFFFFFFFFFFFFFFFBCE6FAADA7179E84F3B9CAC2FC632551
A = -3
B = 0x5AC635D8AA3A93E7B3EBBD55769886BC651D06B0CC53B0F63BCE3C3E27D2604B
G = (0x6B17D1F2E12C4247F8BCE6E563A440F277037D812DEB33A0F4A13945D898C296,
     0x4FE342E2FE1A7F9B8EE7EB4A7C0F9E162BCE33576B315ECECBB6406837BF51F5)


# ---- curve (None is the point at infinity O) -------------------------------------------------------------------------------
def on_curve(pt):
    return pt is None or (pt[1] * pt[1] - (pt[0] ** 3 + A * pt[0] + B)) % P == 0


def neg(pt):
    return None if pt is None else (pt[0], -pt[1] % P)


def add(p1, p2):
    if p1 is None:
        return p2
    if p2 is None:
        return p1
    (x1, y1), (x2, y2) = p1, p2
    if x1 == x2:
        if (y1 + y2) % P == 0:
            return None
        lam = (3 * x1 * x1 + A) * pow(2 * y1, -1, P) % P
    else:
        lam = (y2 - y1) * pow(x2 - x1, -1, P) % P
    x3 = (lam * lam - x1 - x2) % P
    return x3, (lam * (x1 - x3) - y1) % P


def mul(k, pt):
    acc = None
    for bit in bin(k)[2:] if k > 0 else "":
        acc = add(acc, acc)
        if bit == "1":
            acc = add(acc, pt)
    return acc


def lincomb(k1, p1, k2, p2):
    """k1 p1 + k2 p2 by one shared double-and-add (Shamir's trick)"""
    both = add(p1, p2)
    acc = None
    for i in range(max(k1.bit_length(), k2.bit_length()) - 1, -1, -1):
        acc = add(acc, acc)
        b1, b2 = (k1 >> i) & 1, (k2 >> i) & 1
        if b1 and b2:
            acc = add(acc, both)
        elif b1:
            acc = add(acc, p1)
        elif b2:
            acc = add(acc, p2)
    return acc


def sqrt(a):
    """a square root of a mod p (p = 3 mod 4), or None"""
    r = pow(a, (P + 1) // 4, P)
    return r if r * r % P == a % P else None


def lift_x(x):
    y = sqrt((x ** 3 + A * x + B) % P)
    return None if y is None else (x, y)


# ---- P256VERIFY --------------------------------------------------------------------------------------------------------------
def encode(h, r, s, q):
    return b"".join(v.to_bytes(32, "big") for v in (h, r, s, q[0], q[1]))


def decode(inp):
    assert len(inp) == 160
    return [int.from_bytes(inp[32 * i:32 * i + 32], "big") for i in range(5)]


def verify(inp: bytes) -> bool:
    h, r, s, qx, qy = decode(inp)
    if not (1 <= r < N and 1 <= s < N):
        return False
    if qx >= P or qy >= P:
        return False
    q = (qx, qy)
    if not on_curve(q):  # (0, 0) is not on the curve: b != 0
        return False
    z = h % N
    w = pow(s, -1, N)
    rp = lincomb(z * w % N, G, r * w % N, q)
    if rp is None:
        return False
    return rp[0] % N == r


def sign(priv: int, h: int, k: int):
    """ECDSA with a given nonce k -> (r, s) (s as computed, not normalised)"""
    r = mul(k, G)[0] % N
    return r, pow(k, -1, N) * (h % N + r * priv) % N


def high_s(inp: bytes) -> bytes:
    """the same item with s replaced by n - s: both verify (EIP-7951 has no low-s rule)"""
    h, r, s, qx, qy = decode(inp)
    return encode(h, r, N - s, (qx, qy))


# ---- constructions -----------------------------------------------------------------------------------------------------------
def forge(q, u1: int, u2: int):
    """(h, r, s) that verify under the curve point q: R' = u1 G + u2 q, r = x(R') mod n, s = r / u2, h = u1 s"""
    rp = lincomb(u1, G, u2, q)
    r = rp[0] % N
    s = r * pow(u2, -1, N) % N
    return u1 * s % N, r, s


def x_above_n():
    """(valid input, its neighbour with r = x0) for a point R0 whose x0 lies in (n, p): r = x0 - n verifies"""
    x0 = next(x for x in range(N + 1, N + 10000) if lift_x(x) is not None)
    r0 = lift_x(x0)
    r, s, h = x0 - N, 0x1234567, 0x89ABCDEF
    q = mul(pow(r, -1, N), add(mul(s, r0), neg(mul(h, G))))  # Q = r^-1 (s R0 - h G)
    assert q is not None and r + N < P
    return encode(h, r, s, q), encode(h, x0, s, q)


def constructed_cases():
    """[(name, 160-byte input, expected)]: every edge of the rules, each reached by a constructed input"""
    out = []
    d = 0xC0FFEE1234
    q = mul(d, G)
    h, r, s = forge(q, 0x1111, 0x2222)
    out.append(("forged", encode(h, r, s, q), True))
    out.append(("forged_high_s", high_s(encode(h, r, s, q)), True))
    good, neighbour = x_above_n()
    out += [("x_above_n", good, True), ("x_above_n_r_eq_x0", neighbour, False)]
    x2g = mul(2, G)[0] % N
    out.append(("equal_points_2g", encode(x2g, x2g, x2g, G), True))  # u1 = u2 = 1: R' = G + G, the a = -3 doubling
    out.append(("opposite_points", encode(x2g, x2g, x2g, neg(G)), False))  # R' = G - G = O
    ri, si = 0x5EED, 0xB0B
    out.append(("r_prime_infinity", encode(-ri * d % N, ri, si, q), False))  # Q = d G, h = -r d: R' = O
    # forged under keys nobody holds: a small-x point and G itself
    small = next(lift_x(x) for x in range(1, 1000) if lift_x(x) is not None)
    h, r, s = forge(small, 0x77, 0x99)
    out.append(("forged_small_x_key", encode(h, r, s, small), True))
    h, r, s = forge(G, 5, 7)
    out.append(("forged_key_g", encode(h, r, s, G), True))
    return out
