"""Python oracle for ECRECOVER on secp256k1: curve arithmetic over integers, recovery with libsecp256k1's rules (the
default path of the reference's Crypto::secp256k1_ecrecover, recids 2 and 3 included), and a pure-Python keccak256.

recover(sig65, msg32, low_s) -> (status, 32 bytes): status 0 ok, 2 InvalidSignature, 3 RecoveryFailed, 4
InvalidRecoveryId; a failed item gives 32 zero bytes.  The checks run in the order include/b200zk.h documents.
"""
P = 2**256 - 2**32 - 977
N = 0xFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFEBAAEDCE6AF48A03BBFD25E8CD0364141
N_HALF = N // 2
G = (0x79BE667EF9DCBBAC55A06295CE870B07029BFCDB2DCE28D959F2815B16F81798,
     0x483ADA7726A3C4655DA4FBFC0E1108A8FD17B448A68554199C47D08FFB10D4B8)
OK, INVALID_SIGNATURE, RECOVERY_FAILED, INVALID_RECOVERY_ID = 0, 2, 3, 4

# ---- keccak256 (FIPS 202 permutation, written out over 5x5 lanes; original Keccak padding 0x01) ----------------------
_RC = [0x0000000000000001, 0x0000000000008082, 0x800000000000808A, 0x8000000080008000, 0x000000000000808B, 0x0000000080000001,
       0x8000000080008081, 0x8000000000008009, 0x000000000000008A, 0x0000000000000088, 0x0000000080008009, 0x000000008000000A,
       0x000000008000808B, 0x800000000000008B, 0x8000000000008089, 0x8000000000008003, 0x8000000000008002, 0x8000000000000080,
       0x000000000000800A, 0x800000008000000A, 0x8000000080008081, 0x8000000000008080, 0x0000000080000001, 0x8000000080008008]
# rotation offsets r[x][y]
_ROT = [[0, 36, 3, 41, 18], [1, 44, 10, 45, 2], [62, 6, 43, 15, 61], [28, 55, 25, 21, 56], [27, 20, 39, 8, 14]]
_M = (1 << 64) - 1


def _rol(v, s):
    return ((v << s) | (v >> (64 - s))) & _M if s else v


def _keccak_f(a):
    """a[x][y], 64-bit lanes"""
    for rc in _RC:
        c = [a[x][0] ^ a[x][1] ^ a[x][2] ^ a[x][3] ^ a[x][4] for x in range(5)]
        d = [c[(x - 1) % 5] ^ _rol(c[(x + 1) % 5], 1) for x in range(5)]
        a = [[a[x][y] ^ d[x] for y in range(5)] for x in range(5)]
        b = [[0] * 5 for _ in range(5)]
        for x in range(5):
            for y in range(5):
                b[y][(2 * x + 3 * y) % 5] = _rol(a[x][y], _ROT[x][y])
        a = [[b[x][y] ^ (~b[(x + 1) % 5][y] & b[(x + 2) % 5][y]) for y in range(5)] for x in range(5)]
        a[0][0] ^= rc
    return a


def keccak256(data: bytes) -> bytes:
    rate = 136
    m = bytearray(data) + b"\x01"
    m += bytes(-len(m) % rate)
    m[-1] |= 0x80
    a = [[0] * 5 for _ in range(5)]
    for off in range(0, len(m), rate):
        for i in range(rate // 8):
            a[i % 5][i // 5] ^= int.from_bytes(m[off + 8 * i:off + 8 * i + 8], "little")
        a = _keccak_f(a)
    return b"".join(a[i % 5][i // 5].to_bytes(8, "little") for i in range(4))


# ---- curve ----------------------------------------------------------------------------------------------------------------
def on_curve(pt):
    return pt is None or (pt[1] * pt[1] - pt[0] ** 3 - 7) % P == 0


def add(p1, p2):
    if p1 is None:
        return p2
    if p2 is None:
        return p1
    (x1, y1), (x2, y2) = p1, p2
    if x1 == x2:
        if (y1 + y2) % P == 0:
            return None
        lam = 3 * x1 * x1 * pow(2 * y1, -1, P) % P
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


def sqrt(a):
    """a square root of a mod p, or None"""
    r = pow(a, (P + 1) // 4, P)
    return r if r * r % P == a % P else None


def lift_x(x, odd):
    y = sqrt((x ** 3 + 7) % P)
    if y is None:
        return None
    return x, (P - y if (y & 1) != odd else y)


def address_hash(pub) -> bytes:
    return keccak256(pub[0].to_bytes(32, "big") + pub[1].to_bytes(32, "big"))


def address(pub) -> bytes:
    return address_hash(pub)[12:]


def recover_point(sig: bytes, msg: bytes, low_s: bool = False):
    """(status, public key point or None)"""
    assert len(sig) == 65 and len(msg) == 32
    r, s, recid = int.from_bytes(sig[:32], "big"), int.from_bytes(sig[32:64], "big"), sig[64]
    if low_s and s > N_HALF:
        return INVALID_SIGNATURE, None
    if recid > 3:
        return INVALID_RECOVERY_ID, None
    if r >= N or s >= N:
        return INVALID_SIGNATURE, None
    if r == 0 or s == 0:
        return RECOVERY_FAILED, None
    x = r
    if recid & 2:
        if r >= P - N:
            return RECOVERY_FAILED, None
        x = r + N
    R = lift_x(x, recid & 1)
    if R is None:
        return RECOVERY_FAILED, None
    z = int.from_bytes(msg, "big") % N
    ri = pow(r, -1, N)
    q = add(mul(-z * ri % N, G), mul(s * ri % N, R))
    if q is None:
        return RECOVERY_FAILED, None
    return OK, q


def recover(sig: bytes, msg: bytes, low_s: bool = False):
    st, q = recover_point(sig, msg, low_s)
    return st, (address_hash(q) if st == OK else bytes(32))


def sign(priv: int, msg: bytes, k: int):
    """ECDSA with a given nonce k -> 65-byte r | s | recid (s as computed, not normalised)"""
    R = mul(k, G)
    r = R[0] % N
    s = pow(k, -1, N) * (int.from_bytes(msg, "big") + r * priv) % N
    recid = (R[1] & 1) | (2 if R[0] >= N else 0)
    return r.to_bytes(32, "big") + s.to_bytes(32, "big") + bytes([recid])


def verify(pub, sig: bytes, msg: bytes) -> bool:
    """plain ECDSA verification of (r, s) against a public key: an independent check of a recovered key"""
    r, s = int.from_bytes(sig[:32], "big"), int.from_bytes(sig[32:64], "big")
    z, w = int.from_bytes(msg, "big") % N, pow(s, -1, N)
    x = add(mul(z * w % N, G), mul(r * w % N, pub))
    return x is not None and x[0] % N == r


def _sig(r, s, recid):
    return r.to_bytes(32, "big") + s.to_bytes(32, "big") + bytes([recid])


def status_cases():
    """[(name, sig, msg, low_s flag, expected status)]: every status, each reached by a constructed input"""
    msg = bytes(range(1, 33))
    base = sign(0xC0FFEE, msg, 0x1234567)
    r, s, recid = int.from_bytes(base[:32], "big"), int.from_bytes(base[32:64], "big"), base[64]
    lo = low_s(base)
    hi = lo[:32] + (N - int.from_bytes(lo[32:64], "big")).to_bytes(32, "big") + bytes([lo[64] ^ 1])
    no_point = next(x for x in range(1, 1000) if sqrt((x ** 3 + 7) % P) is None)
    rec2 = next(t for t in range(1, 1000) if sqrt(((N + t) ** 3 + 7) % P) is not None)  # x = n + t on the curve, t < p - n
    k = 0xABCDEF0123456789
    kg = mul(k, G)
    assert kg[0] < N
    s_inf = 0x5EED
    z_inf = (s_inf * k % N).to_bytes(32, "big")
    return [
        ("valid", base, msg, False, OK),
        ("low_s_with_flag", lo, msg, True, OK),
        ("high_s_without_flag", hi, msg, False, OK),
        ("high_s_with_flag", hi, msg, True, INVALID_SIGNATURE),
        ("s_half_n_with_flag", _sig(r, N_HALF, recid), msg, True, OK),
        ("s_half_n_plus_1_with_flag", _sig(r, N_HALF + 1, recid), msg, True, INVALID_SIGNATURE),
        ("r_eq_n", _sig(N, s, recid), msg, False, INVALID_SIGNATURE),
        ("s_eq_n", _sig(r, N, recid), msg, False, INVALID_SIGNATURE),
        ("r_max", _sig(2**256 - 1, s, recid), msg, False, INVALID_SIGNATURE),
        ("r_zero", _sig(0, s, recid), msg, False, RECOVERY_FAILED),
        ("s_zero", _sig(r, 0, recid), msg, False, RECOVERY_FAILED),
        ("recid_4", _sig(r, s, 4), msg, False, INVALID_RECOVERY_ID),
        ("recid_255_and_r_eq_n", _sig(N, s, 255), msg, False, INVALID_RECOVERY_ID),
        ("high_s_flag_outranks_recid", _sig(r, N - 1, 9), msg, True, INVALID_SIGNATURE),
        ("x_not_on_curve", _sig(no_point, s, 0), msg, False, RECOVERY_FAILED),
        ("recid_2_recovers", _sig(rec2, s, 2), msg, False, OK),
        ("recid_3_recovers", _sig(rec2, s, 3), msg, False, OK),
        ("recid_2_r_eq_p_minus_n", _sig(P - N, s, 2), msg, False, RECOVERY_FAILED),
        ("recid_3_r_above_p_minus_n", _sig(P - N + 5, s, 3), msg, False, RECOVERY_FAILED),
        ("q_is_identity", _sig(kg[0], s_inf, kg[1] & 1), z_inf, False, RECOVERY_FAILED),
        ("msg_above_n", base[:64] + bytes([base[64]]), (2**256 - 1).to_bytes(32, "big"), False, OK),
    ]


def low_s(sig: bytes) -> bytes:
    """the same signature with s replaced by n - s when s > n/2 (recid's parity flips), as a transaction carries it"""
    s = int.from_bytes(sig[32:64], "big")
    if s <= N_HALF:
        return sig
    return sig[:32] + (N - s).to_bytes(32, "big") + bytes([sig[64] ^ 1])
