"""oracle/bls_ref.py -- TEST INFRASTRUCTURE ONLY: pure-Python big-integer BLS12-381 G1 (y^2 = x^3 + 4 over Fp) with the
48-byte compressed ZCash / IETF encoding, restated from the published curve parameters (draft-irtf-cfrg-pairing-friendly-
curves, EIP-2537 / EIP-4844): what c-kzg 's blob_to_kzg_commitment computes, which ethrex reaches through
/root/reference/crates/common/crypto/kzg.rs:259-272.  "parity unpinned": the reference tree holds neither the 4096-point
trusted setup (it ships inside the c-kzg / kzg-rs crates) nor a BLS12-381 G1 vector computed under it -- the commitments in
/root/reference/crates/common/types/blobs_bundle.rs:430-485 are mainnet values under that setup.  What IS pinned here: the
generator and the field / group orders (checked against each other: r * G = identity), and the encoding of the identity and
of the generator, which are public constants.  Only tests/ may import this module."""
P = 0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab
R = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001
G1 = (0x17f1d3a73197d7942695638c4fa9ac0fc3688c4f9774b905a14e3a3f171bac586c55e83ff97a1aeffb3af00adb22c6bb,
      0x08b3f481e3aaa0f1a09e30ed741d8ae4fcf5e095d5d00af600db18cb2c04b3edd03cc744a2888ae40caa232946c5e7e1)
# compressed generator, a public constant (e.g. the first G1 point of every BLS12-381 test suite)
G1_COMPRESSED = bytes.fromhex("97f1d3a73197d7942695638c4fa9ac0fc3688c4f9774b905a14e3a3f171bac586c55e83ff97a1aeffb3af00adb22c6bb")
FIELD_ELEMENTS_PER_BLOB = 4096
# primitive 4096-th root of unity of the scalar field: 7^((r-1)/4096) (c-kzg: SCALE2_ROOT_OF_UNITY[12])
ROOT_4096 = pow(7, (R - 1) // FIELD_ELEMENTS_PER_BLOB, R)


def add(p, q):
    if p is None:
        return q
    if q is None:
        return p
    (x1, y1), (x2, y2) = p, q
    if x1 == x2:
        if (y1 + y2) % P == 0:
            return None
        lam = 3 * x1 * x1 * pow(2 * y1, -1, P) % P
    else:
        lam = (y2 - y1) * pow(x2 - x1, -1, P) % P
    x3 = (lam * lam - x1 - x2) % P
    return x3, (lam * (x1 - x3) - y1) % P


def mul(k, p):
    k %= R
    acc = None
    while k:
        if k & 1:
            acc = add(acc, p)
        p = add(p, p)
        k >>= 1
    return acc


def on_curve(p):
    return p is None or (p[1] * p[1] - p[0] ** 3 - 4) % P == 0


def compress(p) -> bytes:
    if p is None:
        return bytes([0xC0]) + bytes(47)
    x, y = p
    b = bytearray(x.to_bytes(48, "big"))
    b[0] |= 0x80 | (0x20 if y > (P - 1) // 2 else 0)
    return bytes(b)


def decompress(b: bytes):
    assert len(b) == 48 and b[0] & 0x80
    if b[0] & 0x40:
        return None
    x = int.from_bytes(b, "big") & ((1 << 381) - 1)
    y = pow((x ** 3 + 4) % P, (P + 1) // 4, P)
    assert (y * y - x ** 3 - 4) % P == 0, "not on the curve"
    if (y > (P - 1) // 2) != bool(b[0] & 0x20):
        y = P - y
    return x, y


def uncompressed(p) -> bytes:
    if p is None:
        return bytes([0x40]) + bytes(95)
    return p[0].to_bytes(48, "big") + p[1].to_bytes(48, "big")


def bit_reverse(i: int, bits: int) -> int:
    return int(format(i, f"0{bits}b")[::-1], 2)


def lagrange_setup_scalars(tau: int, n: int = FIELD_ELEMENTS_PER_BLOB):
    """L_i(tau) for the size-n domain in BIT-REVERSED order (c-kzg's g1_lagrange_brp): the i-th entry belongs to the root
    w^brp(i).  L_j(tau) = w^j (tau^n - 1) / (n (tau - w^j))."""
    bits = n.bit_length() - 1
    w = pow(7, (R - 1) // n, R)
    zt, ninv = (pow(tau, n, R) - 1) % R, pow(n, -1, R)
    out = []
    for i in range(n):
        wj = pow(w, bit_reverse(i, bits), R)
        out.append(wj * zt % R * ninv % R * pow((tau - wj) % R, -1, R) % R)
    return out


def msm(scalars, points):
    acc = None
    for s, p in zip(scalars, points):
        acc = add(acc, mul(s, p))
    return acc


# ---- fast fixed-base multiples of the generator (Jacobian accumulation over a table of 2^i G): building a synthetic
# 4096-point setup with `mul` (affine, one inversion per step) would take minutes
_POW2 = None


def _pow2_table():
    global _POW2
    if _POW2 is None:
        t, p = [], G1
        for _ in range(255):
            t.append(p)
            p = add(p, p)
        _POW2 = t
    return _POW2


def _jac_add_mixed(X1, Y1, Z1, x2, y2):
    if Z1 == 0:
        return x2, y2, 1
    Z1Z1 = Z1 * Z1 % P
    U2, S2 = x2 * Z1Z1 % P, y2 * Z1 * Z1Z1 % P
    H, r = (U2 - X1) % P, (S2 - Y1) % P
    if H == 0:
        if r == 0:  # doubling (never with distinct table entries, kept for completeness)
            a = add((x2, y2), (x2, y2))
            return a[0], a[1], 1
        return 0, 1, 0
    HH = H * H % P
    HHH, V = H * HH % P, X1 * HH % P
    X3 = (r * r - HHH - 2 * V) % P
    return X3, (r * (V - X3) - Y1 * HHH) % P, Z1 * H % P


def chain(n: int, k: int, d: int, block: int = 4096):
    """Synthetic bases P_i = (k + i*d) * G, i < n, as n x 96 bytes uncompressed big-endian (identity: the 0x40 form) --
    what bls12_381_g1_bases_upload(..., flags=0) takes.  Every base is a known multiple of G, so an MSM over them has the
    closed form ((sum_i s_i (k + i d)) mod r) * G: one scalar multiplication, whatever n.  Built by Jacobian mixed
    additions of D = d * G, normalised a block at a time with one inversion per block (Montgomery's trick)."""
    k0, dd = generator_multiples([k, d])
    out = bytearray()
    X, Y, Z = (k0[0], k0[1], 1) if k0 is not None else (0, 1, 0)
    for lo in range(0, n, block):
        jac = []
        for _ in range(min(block, n - lo)):
            jac.append((X, Y, Z))
            if dd is not None:
                X, Y, Z = _jac_add_mixed(X, Y, Z, *dd)
        prefix, acc = [], 1
        for _, _, z in jac:
            prefix.append(acc)
            if z:
                acc = acc * z % P
        inv = pow(acc, -1, P)
        aff = [None] * len(jac)
        for j in range(len(jac) - 1, -1, -1):
            x, y, z = jac[j]
            if z:
                zi = inv * prefix[j] % P
                inv = inv * z % P
                zi2 = zi * zi % P
                aff[j] = (x * zi2 % P, y * zi2 * zi % P)
        for p in aff:
            out += uncompressed(p)
    return bytes(out)


def generator_multiples(scalars):
    """[s * G for s in scalars] (affine, None for the identity)"""
    tab = _pow2_table()
    out = []
    for s in scalars:
        s %= R
        X, Y, Z = 0, 1, 0
        i = 0
        while s:
            if s & 1:
                X, Y, Z = _jac_add_mixed(X, Y, Z, *tab[i])
            s >>= 1
            i += 1
        if Z == 0:
            out.append(None)
        else:
            zi = pow(Z, -1, P)
            out.append((X * zi * zi % P, Y * zi * zi * zi % P))
    return out
