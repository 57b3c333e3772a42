"""EIP-2537 map-to-curve reference -- TEST INFRASTRUCTURE ONLY (the library's is ethrex_b200/csrc/bls_map.cu).

RFC 9380 as the bls12_381 crate implements it: map_to_curve_simple_swu (section 6.6.2) on the isogenous curve E',
iso_map (6.6.3) onto E, then clear_cofactor (section 7), with the BLS12-381 parameters of 8.8.1 (G1) and 8.8.2 (G2).
Written in affine big-integer arithmetic over the independent oracles (oracle/bls_ref.py for G1, tests/bls_pairing_ref.py
for G2), deliberately unlike the device's Montgomery / XYZZ code.  G2's clear_cofactor is here both ways: the psi form of
RFC Appendix G.3, which the device uses, and the plain scalar h_eff, which defines it.

The isogeny tables are RFC Appendix E.2 (G1, 11-isogeny) and E.3 (G2, 3-isogeny), coefficients k_(i,0), k_(i,1), ... in
ascending powers of x; x_den and y_den are monic and their leading 1 is not listed.  tests/golden/make_bls12_map_constants.py
checks them against the curves (G1) and re-derives them from the reference's one vector (G2)."""
import bls_pairing_ref as B
import bls_ref as bls

P, R = B.P, B.R
Z_ABS = 0xD201000000010000  # |z|, the BLS parameter z = -0xd201000000010000
H_EFF_G1 = 0xD201000000010001  # 1 - z
H_EFF_G2 = int("bc69f08f2ee75b3584c6a0ea91b352888e2a8e9145ad7689986ff031508ffe1329c2f178731db956d82bf015d1212b02ec0ec69d7477c1ae"
               "954cbc06689f6a359894c0adebbf6b4e8020005aaa95551", 16)

# ---- G1: E': y^2 = x^3 + A' x + B' over Fp, Z = 11 (RFC 8.8.1)
G1_A = 0x144698a3b8e9433d693a02c96d4982b0ea985383ee66a8d8e8981aefd881ac98936f8da0e0f97f5cf428082d584c1d
G1_B = 0x12e2908d11688030018b12e8753eee3b2016c1f0f24f4070a0b9c14fcef35ef55a23215a316ceaa5d1cc48e98e172be0
G1_Z = 11
# RFC Appendix E.2
G1_XNUM = [
    0x11a05f2b1e833340b809101dd99815856b303e88a2d7005ff2627b56cdb4e2c85610c2d5f2e62d6eaeac1662734649b7,
    0x17294ed3e943ab2f0588bab22147a81c7c17e75b2f6a8417f565e33c70d1e86b4838f2a6f318c356e834eef1b3cb83bb,
    0xd54005db97678ec1d1048c5d10a9a1bce032473295983e56878e501ec68e25c958c3e3d2a09729fe0179f9dac9edcb0,
    0x1778e7166fcc6db74e0609d307e55412d7f5e4656a8dbf25f1b33289f1b330835336e25ce3107193c5b388641d9b6861,
    0xe99726a3199f4436642b4b3e4118e5499db995a1257fb3f086eeb65982fac18985a286f301e77c451154ce9ac8895d9,
    0x1630c3250d7313ff01d1201bf7a74ab5db3cb17dd952799b9ed3ab9097e68f90a0870d2dcae73d19cd13c1c66f652983,
    0xd6ed6553fe44d296a3726c38ae652bfb11586264f0f8ce19008e218f9c86b2a8da25128c1052ecaddd7f225a139ed84,
    0x17b81e7701abdbe2e8743884d1117e53356de5ab275b4db1a682c62ef0f2753339b7c8f8c8f475af9ccb5618e3f0c88e,
    0x80d3cf1f9a78fc47b90b33563be990dc43b756ce79f5574a2c596c928c5d1de4fa295f296b74e956d71986a8497e317,
    0x169b1f8e1bcfa7c42e0c37515d138f22dd2ecb803a0c5c99676314baf4bb1b7fa3190b2edc0327797f241067be390c9e,
    0x10321da079ce07e272d8ec09d2565b0dfa7dccdde6787f96d50af36003b14866f69b771f8c285decca67df3f1605fb7b,
    0x6e08c248e260e70bd1e962381edee3d31d79d7e22c837bc23c0bf1bc24c6b68c24b1b80b64d391fa9c8ba2e8ba2d229,
]
G1_XDEN = [
    0x8ca8d548cff19ae18b2e62f4bd3fa6f01d5ef4ba35b48ba9c9588617fc8ac62b558d681be343df8993cf9fa40d21b1c,
    0x12561a5deb559c4348b4711298e536367041e8ca0cf0800c0126c2588c48bf5713daa8846cb026e9e5c8276ec82b3bff,
    0xb2962fe57a3225e8137e629bff2991f6f89416f5a718cd1fca64e00b11aceacd6a3d0967c94fedcfcc239ba5cb83e19,
    0x3425581a58ae2fec83aafef7c40eb545b08243f16b1655154cca8abc28d6fd04976d5243eecf5c4130de8938dc62cd8,
    0x13a8e162022914a80a6f1d5f43e7a07dffdfc759a12062bb8d6b44e833b306da9bd29ba81f35781d539d395b3532a21e,
    0xe7355f8e4e667b955390f7f0506c6e9395735e9ce9cad4d0a43bcef24b8982f7400d24bc4228f11c02df9a29f6304a5,
    0x772caacf16936190f3e0c63e0596721570f5799af53a1894e2e073062aede9cea73b3538f0de06cec2574496ee84a3a,
    0x14a7ac2a9d64a8b230b3f5b074cf01996e7f63c21bca68a81996e1cdf9822c580fa5b9489d11e2d311f7d99bbdcc5a5e,
    0xa10ecf6ada54f825e920b3dafc7a3cce07f8d1d7161366b74100da67f39883503826692abba43704776ec3a79a1d641,
    0x95fc13ab9e92ad4476d6e3eb3a56680f682b4ee96f7d03776df533978f31c1593174e4b4b7865002d6384d168ecdd0a,
]
G1_YNUM = [
    0x90d97c81ba24ee0259d1f094980dcfa11ad138e48a869522b52af6c956543d3cd0c7aee9b3ba3c2be9845719707bb33,
    0x134996a104ee5811d51036d776fb46831223e96c254f383d0f906343eb67ad34d6c56711962fa8bfe097e75a2e41c696,
    0xcc786baa966e66f4a384c86a3b49942552e2d658a31ce2c344be4b91400da7d26d521628b00523b8dfe240c72de1f6,
    0x1f86376e8981c217898751ad8746757d42aa7b90eeb791c09e4a3ec03251cf9de405aba9ec61deca6355c77b0e5f4cb,
    0x8cc03fdefe0ff135caf4fe2a21529c4195536fbe3ce50b879833fd221351adc2ee7f8dc099040a841b6daecf2e8fedb,
    0x16603fca40634b6a2211e11db8f0a6a074a7d0d4afadb7bd76505c3d3ad5544e203f6326c95a807299b23ab13633a5f0,
    0x4ab0b9bcfac1bbcb2c977d027796b3ce75bb8ca2be184cb5231413c4d634f3747a87ac2460f415ec961f8855fe9d6f2,
    0x987c8d5333ab86fde9926bd2ca6c674170a05bfe3bdd81ffd038da6c26c842642f64550fedfe935a15e4ca31870fb29,
    0x9fc4018bd96684be88c9e221e4da1bb8f3abd16679dc26c1e8b6e6a1f20cabe69d65201c78607a360370e577bdba587,
    0xe1bba7a1186bdb5223abde7ada14a23c42a0ca7915af6fe06985e7ed1e4d43b9b3f7055dd4eba6f2bafaaebca731c30,
    0x19713e47937cd1be0dfd0b8f1d43fb93cd2fcbcb6caf493fd1183e416389e61031bf3a5cce3fbafce813711ad011c132,
    0x18b46a908f36f6deb918c143fed2edcc523559b8aaf0c2462e6bfe7f911f643249d9cdf41b44d606ce07c8a4d0074d8e,
    0xb182cac101b9399d155096004f53f447aa7b12a3426b08ec02710e807b4633f06c851c1919211f20d4c04f00b971ef8,
    0x245a394ad1eca9b72fc00ae7be315dc757b3b080d4c158013e6632d3c40659cc6cf90ad1c232a6442d9d3f5db980133,
    0x5c129645e44cf1102a159f748c4a3fc5e673d81d7e86568d9ab0f5d396a7ce46ba1049b6579afb7866b1e715475224b,
    0x15e6be4e990f03ce4ea50b3b42df2eb5cb181d8f84965a3957add4fa95af01b2b665027efec01c7704b456be69c8b604,
]
G1_YDEN = [
    0x16112c4c3a9c98b252181140fad0eae9601a6de578980be6eec3232b5be72e7a07f3688ef60c206d01479253b03663c1,
    0x1962d75c2381201e1a0cbd6c43c348b885c84ff731c4d59ca4a10356f453e01f78a4260763529e3532f6102c2e49a03d,
    0x58df3306640da276faaae7d6e8eb15778c4855551ae7f310c35a5dd279cd2eca6757cd636f96f891e2538b53dbf67f2,
    0x16b7d288798e5395f20d23bf89edb4d1d115c5dbddbcd30e123da489e726af41727364f2c28297ada8d26d98445f5416,
    0xbe0e079545f43e4b00cc912f8228ddcc6d19c9f0f69bbb0542eda0fc9dec916a20b15dc0fd2ededda39142311a5001d,
    0x8d9e5297186db2d9fb266eaac783182b70152c65550d881c5ecd87b6f0f5a6449f38db9dfa9cce202c6477faaf9b7ac,
    0x166007c08a99db2fc3ba8734ace9824b5eecfdfa8d0cf8ef5dd365bc400a0051d5fa9c01a58b1fb93d1a1399126a775c,
    0x16a3ef08be3ea7ea03bcddfabba6ff6ee5a4375efa1f4fd7feb34fd206357132b920f5b00801dee460ee415a15812ed9,
    0x1866c8ed336c61231a1be54fd1d74cc4f9fb0ce4c6af5920abc5750c4bf39b4852cfe2f7bb9248836b233d9d55535d4a,
    0x167a55cda70a6e1cea820597d94a84903216f763e13d87bb5308592e7ea7d4fbc7385ea3d529b35e346ef48bb8913f55,
    0x4d2f259eea405bd48f010a01ad2911d9c6dd039bb61a6290e591b36e636a5c871a5c29f4f83060400f8b49cba8f6aa8,
    0xaccbb67481d033ff5852c1e48c50c477f94ff8aefce42d28c0f9a88cea7913516f968986f7ebbea9684b529e2561092,
    0xad6b9514c767fe3c3613144b45f1496543346d98adf02267d5ceef9a00d9b8693000763e3b90ac11e99b138573345cc,
    0x2660400eb2e4f3b628bdd0d53cd76f2bf565b94e72927c1cb748df27942480e420517bd8714cc80d1fadc1326ed06f7,
    0xe0fa1d816ddc03e6b24255e0d7819c171c40f65e273b853324efcd6356caa205ca2f570f13497804415473a1d634b8f,
]

# ---- G2: E2': y^2 = x^3 + A' x + B' over Fp2, A' = 240 i, B' = 1012 (1 + i), Z = -(2 + i) (RFC 8.8.2)
G2_A = (0, 240)
G2_B = (1012, 1012)
G2_Z = (P - 2, P - 1)
# RFC Appendix E.3, (c0, c1) pairs
G2_XNUM = [
    (0x5c759507e8e333ebb5b7a9a47d7ed8532c52d39fd3a042a88b58423c50ae15d5c2638e343d9c71c6238aaaaaaaa97d6,
     0x5c759507e8e333ebb5b7a9a47d7ed8532c52d39fd3a042a88b58423c50ae15d5c2638e343d9c71c6238aaaaaaaa97d6),
    (0x0,
     0x11560bf17baa99bc32126fced787c88f984f87adf7ae0c7f9a208c6b4f20a4181472aaa9cb8d555526a9ffffffffc71a),
    (0x11560bf17baa99bc32126fced787c88f984f87adf7ae0c7f9a208c6b4f20a4181472aaa9cb8d555526a9ffffffffc71e,
     0x8ab05f8bdd54cde190937e76bc3e447cc27c3d6fbd7063fcd104635a790520c0a395554e5c6aaaa9354ffffffffe38d),
    (0x171d6541fa38ccfaed6dea691f5fb614cb14b4e7f4e810aa22d6108f142b85757098e38d0f671c7188e2aaaaaaaa5ed1,
     0x0),
]
G2_XDEN = [
    (0x0,
     0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaa63),
    (0xc,
     0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaa9f),
]
G2_YNUM = [
    (0x1530477c7ab4113b59a4c18b076d11930f7da5d4a07f649bf54439d87d27e500fc8c25ebf8c92f6812cfc71c71c6d706,
     0x1530477c7ab4113b59a4c18b076d11930f7da5d4a07f649bf54439d87d27e500fc8c25ebf8c92f6812cfc71c71c6d706),
    (0x0,
     0x5c759507e8e333ebb5b7a9a47d7ed8532c52d39fd3a042a88b58423c50ae15d5c2638e343d9c71c6238aaaaaaaa97be),
    (0x11560bf17baa99bc32126fced787c88f984f87adf7ae0c7f9a208c6b4f20a4181472aaa9cb8d555526a9ffffffffc71c,
     0x8ab05f8bdd54cde190937e76bc3e447cc27c3d6fbd7063fcd104635a790520c0a395554e5c6aaaa9354ffffffffe38f),
    (0x124c9ad43b6cf79bfbf7043de3811ad0761b0f37a1e26286b0e977c69aa274524e79097a56dc4bd9e1b371c71c718b10,
     0x0),
]
G2_YDEN = [
    (0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffa8fb,
     0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffa8fb),
    (0x0,
     0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffa9d3),
    (0x12,
     0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaa99),
]
G1_TABLES = (G1_XNUM, G1_XDEN, G1_YNUM, G1_YDEN)
G2_TABLES = (G2_XNUM, G2_XDEN, G2_YNUM, G2_YDEN)


# ---- the two coordinate fields behind one interface
class Fp:
    zero, one = 0, 1
    add = staticmethod(lambda a, b: (a + b) % P)
    sub = staticmethod(lambda a, b: (a - b) % P)
    mul = staticmethod(lambda a, b: a * b % P)
    neg = staticmethod(lambda a: -a % P)
    inv0 = staticmethod(lambda a: pow(a, P - 2, P))  # inv0(0) = 0

    @staticmethod
    def sqrt(a):
        y = pow(a, (P + 1) // 4, P)
        return y if y * y % P == a else None

    @staticmethod
    def sgn0(a):
        return a & 1


class Fp2:
    zero, one = (0, 0), (1, 0)
    add, sub, mul, neg = staticmethod(B.f2_add), staticmethod(B.f2_sub), staticmethod(B.f2_mul), staticmethod(B.f2_neg)
    sqrt = staticmethod(B.f2_sqrt)

    @staticmethod
    def inv0(a):
        return (0, 0) if a == (0, 0) else B.f2_inv(a)

    @staticmethod
    def sgn0(a):
        return (a[0] & 1) | (a[0] == 0 and a[1] & 1)


def poly(F, coeffs, x, monic=False):
    """Horner, coefficients in ascending powers; monic appends the unlisted leading 1"""
    acc = F.one if monic else F.zero
    for c in reversed(coeffs):
        acc = F.add(F.mul(acc, x), c)
    return acc


def sswu(F, A, Bc, Z, u):
    """map_to_curve_simple_swu (RFC 9380 6.6.2) onto y^2 = x^3 + A x + B, straight-line form"""
    g = lambda x: F.add(F.mul(F.add(F.mul(x, x), A), x), Bc)  # noqa: E731
    zu2 = F.mul(Z, F.mul(u, u))
    tv1 = F.inv0(F.add(F.mul(zu2, zu2), zu2))
    if tv1 == F.zero:
        x1 = F.mul(Bc, F.inv0(F.mul(Z, A)))
    else:
        x1 = F.mul(F.neg(F.mul(Bc, F.inv0(A))), F.add(F.one, tv1))
    y = F.sqrt(g(x1))
    x = x1
    if y is None:
        x = F.mul(zu2, x1)
        y = F.sqrt(g(x))
    if F.sgn0(u) != F.sgn0(y):
        y = F.neg(y)
    return x, y


def iso_map(F, tables, pt):
    """(x_num / x_den, y y_num / y_den); the identity (None) where a denominator vanishes"""
    xnum, xden, ynum, yden = tables
    x, y = pt
    xd, yd = poly(F, xden, x, monic=True), poly(F, yden, x, monic=True)
    if xd == F.zero or yd == F.zero:
        return None
    return F.mul(poly(F, xnum, x), F.inv0(xd)), F.mul(y, F.mul(poly(F, ynum, x), F.inv0(yd)))


def _mul(add, k, p):
    """k p by double-and-add, k not reduced (correct outside the subgroup)"""
    acc = None
    while k:
        if k & 1:
            acc = add(acc, p)
        p = add(p, p)
        k >>= 1
    return acc


def _g1_neg(p):
    return None if p is None else (p[0], -p[1] % P)


# psi = Frobenius conjugated by the twist: psi(x, y) = (c_x conj(x), c_y conj(y)), c_x = 1/(1+i)^((p-1)/3), c_y = 1/(1+i)^((p-1)/2)
PSI_CX = B.f2_inv(B.f2_pow((1, 1), (P - 1) // 3))
PSI_CY = B.f2_inv(B.f2_pow((1, 1), (P - 1) // 2))


def psi(q):
    if q is None:
        return None
    (x0, x1), (y0, y1) = q
    return B.f2_mul(PSI_CX, (x0, -x1 % P)), B.f2_mul(PSI_CY, (y0, -y1 % P))


def g2_mul_z(q):
    """z q, z = -|z| negative"""
    return B.g2_neg(_mul(B.g2_add, Z_ABS, q))


def clear_cofactor_g2_psi(q):
    """RFC 9380 Appendix G.3: [z^2 - z - 1] q + [z - 1] psi(q) + psi^2(2 q)"""
    add, neg = B.g2_add, B.g2_neg
    t1 = g2_mul_z(q)
    t2 = psi(q)
    t3 = psi(psi(add(q, q)))
    t3 = add(t3, neg(t2))
    t2 = g2_mul_z(add(t1, t2))
    t3 = add(add(t3, t2), neg(t1))
    return add(t3, neg(q))


def clear_cofactor_g2_scalar(q):
    return _mul(B.g2_add, H_EFF_G2, q)




def map_to_g1(u):
    return _mul(bls.add, H_EFF_G1, iso_map(Fp, G1_TABLES, sswu(Fp, G1_A, G1_B, G1_Z, u % P)))


def map_to_g2(u):
    return clear_cofactor_g2_psi(iso_map(Fp2, G2_TABLES, sswu(Fp2, G2_A, G2_B, G2_Z, (u[0] % P, u[1] % P))))


# ---- the precompile's bytes: 64-byte padded field elements in, padded EIP-2537 points out, with the device's status
def _fp(b: bytes):
    v = int.from_bytes(b[16:64], "big")
    return v if b[:16] == bytes(16) and v < P else None


def map_fp_to_g1_bytes(data: bytes):
    """(128-byte output, status): 0 ok, 1 identity, 2 nonzero padding or a value >= p (output all zero)"""
    u = _fp(data)
    if u is None:
        return bytes(128), 2
    pt = map_to_g1(u)
    return B.g1_eip2537(pt), (1 if pt is None else 0)


def map_fp2_to_g2_bytes(data: bytes):
    c0, c1 = _fp(data[:64]), _fp(data[64:128])
    if c0 is None or c1 is None:
        return bytes(256), 2
    pt = map_to_g2((c0, c1))
    return B.g2_eip2537(pt), (1 if pt is None else 0)


def fp64(v: int) -> bytes:
    return B.fp64(v)


def fp2_64(u) -> bytes:
    return B.fp64(u[0]) + B.fp64(u[1])
