"""Groth16 from circom artifacts: a snarkjs `.zkey` loaded once into HBM, each `.wtns` witness proved in one call.

The two files risc0-groth16's shrink-wrap hands its prover (the proving key, the witness circom-witnesscalc computed),
taken byte for byte; formats and the proof they give are stated in include/b200zk.h (b200zk_groth16_zkey_*).  The
sparse evaluation of the constraint rows, the NTTs onto the odd coset, the MSMs and the blinding all run in
libb200zk.so; Python passes bytes.
"""
from __future__ import annotations

import ctypes as C
import os

from . import _ffi as F
from .context import _current_stream_ptr, _host_ptr
from .groth16 import Groth16Verifier, random_scalar


def _bytes(src) -> bytes:
    """file contents from bytes-like data or a path"""
    if isinstance(src, (str, os.PathLike)):
        with open(src, "rb") as f:
            return f.read()
    return bytes(src)


class ZkeyProver:
    """`ZkeyProver(ctx, zkey, precompute=True)`: zkey is the .zkey file's bytes or its path.  `precompute` builds the
    window tables of the five columns (faster MSMs, about 13x the columns' memory)."""

    def __init__(self, ctx, zkey, precompute: bool = True):
        data = _bytes(zkey)
        ptr, keep = _host_ptr(data)
        h = C.c_uint64()
        ctx._check(F.lib.b200zk_groth16_zkey_load(ctx._h, ptr, len(data), 1 if precompute else 0, C.byref(h)), "b200zk_groth16_zkey_load")
        del keep
        self.ctx, self.key = ctx, h.value
        try:
            nv, npub, log_n = C.c_uint32(), C.c_uint32(), C.c_uint32()
            ctx._check(F.lib.b200zk_groth16_zkey_info(ctx._h, self.key, C.byref(nv), C.byref(npub), C.byref(log_n), None, 0), "b200zk_groth16_zkey_info")
            self.n_vars, self.n_public, self.log_n = nv.value, npub.value, log_n.value
            vk = C.create_string_buffer(448 + 64 * (self.n_public + 1))
            ctx._check(F.lib.b200zk_groth16_zkey_info(ctx._h, self.key, None, None, None, vk, len(vk.raw)), "b200zk_groth16_zkey_info")
            self.vk = vk.raw  # alpha1 | beta2 | gamma2 | delta2 | IC, EIP-196/197 bytes
        except BaseException:
            self.close()  # a prover that failed to construct leaves no key behind
            raise

    def verifier(self) -> Groth16Verifier:
        """the Groth16 verifier of this key (public inputs: signals 1..nPublic of the witness)"""
        v = self.vk
        ic = [v[448 + 64 * i: 512 + 64 * i] for i in range(self.n_public + 1)]
        return Groth16Verifier(self.ctx, v[:64], v[64:192], v[192:320], v[320:448], ic)

    def prove(self, wtns, r: int | None = None, s: int | None = None) -> bytes:
        """-> proof A (64) | B (128) | C (64) of the .wtns witness (bytes or a path), blinded with r and s (each in
        [0, group order); None = a fresh draw of `random_scalar`).  ONE call of the C ABI (b200zk_groth16_zkey_prove)."""
        if self.key is None:
            raise ValueError("ZkeyProver is closed")
        data = _bytes(wtns)
        r = random_scalar() if r is None else r
        s = random_scalar() if s is None else s
        if not (0 <= r < 1 << 256 and 0 <= s < 1 << 256):
            raise ValueError("r and s must be 256-bit non-negative integers")
        ptr, keep = _host_ptr(data)
        rb = C.create_string_buffer(int(r).to_bytes(32, "little"), 32)
        sb = C.create_string_buffer(int(s).to_bytes(32, "little"), 32)
        proof = C.create_string_buffer(256)
        self.ctx._check(F.lib.b200zk_groth16_zkey_prove(self.ctx._h, self.key, ptr, len(data), rb, sb, _current_stream_ptr(self.ctx.device), proof),
                        "b200zk_groth16_zkey_prove")
        del keep
        return proof.raw

    def close(self):
        if self.key is not None:
            self.ctx._check(F.lib.b200zk_groth16_zkey_free(self.ctx._h, self.key), "b200zk_groth16_zkey_free")
            self.key = None


# ---- PLONK (snarkjs 0.7) ------------------------------------------------------------------------------------------------
R_MOD = 0x30644E72E131A029B85045B68181585D2833E84879B9709143E1F593F0000001
P_MOD = 0x30644E72E131A029B85045B68181585D97816A916871CA8D3C208C16D87CFD47
G2_ONE = bytes.fromhex(  # the BN254 G2 generator, EIP-197 x_im | x_re | y_im | y_re
    "198e9393920d483a7260bfb731fb5d25f1aa493335a9e71297e485b7aef312c2"
    "1800deef121f1e76426a00665e5c4479674322d4f75edadd46debd5cd992f6ed"
    "090689d0585ff075ec9e99ad690c3395bc4b313370b38ef355acdadcd122975b"
    "12c85ea5db8c6deb4aab71808dcb408fe3d1e7690c43d37b4ce6cc0166fa7daa")

_KECCAK_RC = [0x0000000000000001, 0x0000000000008082, 0x800000000000808A, 0x8000000080008000, 0x000000000000808B, 0x0000000080000001,
              0x8000000080008081, 0x8000000000008009, 0x000000000000008A, 0x0000000000000088, 0x0000000080008009, 0x000000008000000A,
              0x000000008000808B, 0x800000000000008B, 0x8000000000008089, 0x8000000000008003, 0x8000000000008002, 0x8000000000000080,
              0x000000000000800A, 0x800000008000000A, 0x8000000080008081, 0x8000000000008080, 0x0000000080000001, 0x8000000080008008]
_KECCAK_ROT = [[0, 36, 3, 41, 18], [1, 44, 10, 45, 2], [62, 6, 43, 15, 61], [28, 55, 25, 21, 56], [27, 20, 39, 8, 14]]
_M64 = (1 << 64) - 1


def keccak256(data: bytes) -> bytes:
    """Keccak-256 (original padding 0x01; hashlib's sha3_256 pads with 0x06): the PLONK transcript's hash"""
    rol = lambda v, s: ((v << s) | (v >> (64 - s))) & _M64 if s else v
    m = bytearray(data) + b"\x01"
    m += bytes(-len(m) % 136)
    m[-1] |= 0x80
    a = [[0] * 5 for _ in range(5)]
    for off in range(0, len(m), 136):
        for i in range(17):
            a[i % 5][i // 5] ^= int.from_bytes(m[off + 8 * i:off + 8 * i + 8], "little")
        for rc in _KECCAK_RC:
            c = [a[x][0] ^ a[x][1] ^ a[x][2] ^ a[x][3] ^ a[x][4] for x in range(5)]
            d = [c[(x - 1) % 5] ^ rol(c[(x + 1) % 5], 1) for x in range(5)]
            b = [[0] * 5 for _ in range(5)]
            for x in range(5):
                for y in range(5):
                    b[y][(2 * x + 3 * y) % 5] = rol(a[x][y] ^ d[x], _KECCAK_ROT[x][y])
            a = [[b[x][y] ^ (~b[(x + 1) % 5][y] & b[(x + 2) % 5][y]) for y in range(5)] for x in range(5)]
            a[0][0] ^= rc
    return b"".join(a[i % 5][i // 5].to_bytes(8, "little") for i in range(4))


def _challenge(data: bytes) -> int:
    return int.from_bytes(keccak256(data), "big") % R_MOD


def _be(v: int) -> bytes:
    return (v % R_MOD).to_bytes(32, "big")


class PlonkVerifier:
    """snarkjs 0.7's plonk_verify.js on the device: the challenges (u = H(Wxi, Wxiw) included) in Python, the G1
    combinations as two MSMs, and the final check e(-A1, X_2) e(B1, [1]2) = 1 as one two-pair check through
    b200zk_bn254_pairing_check_batch.  vk: the 736 bytes of b200zk_plonk_zkey_info."""

    def __init__(self, ctx, vk: bytes, n_public: int, log_n: int):
        if len(vk) != 736:
            raise ValueError("a PLONK verifying key is 736 bytes")
        self.ctx, self.vk, self.n_public, self.log_n = ctx, bytes(vk), n_public, log_n

    def verify(self, proof: bytes, public_inputs) -> bool:
        if len(proof) != 768 or len(public_inputs) != self.n_public:
            raise ValueError("proof must be 768 bytes and carry nPublic public inputs")
        pts = [proof[64 * i:64 * i + 64] for i in range(9)]
        evs = [int.from_bytes(proof[576 + 32 * i:608 + 32 * i], "big") for i in range(6)]
        if any(int.from_bytes(p[:32], "big") >= P_MOD or int.from_bytes(p[32:], "big") >= P_MOD for p in pts):
            return False
        if any(e >= R_MOD for e in evs) or any((not isinstance(x, int)) or not 0 <= x < R_MOD for x in public_inputs):
            return False
        vk = self.vk
        A, B, Cc, Z, T1, T2, T3, Wxi, Wxiw = pts
        ea, eb, ec, es1, es2, ezw = evs
        Qm, Ql, Qr, Qo, Qc, S1, S2, S3 = (vk[64 * i:64 * i + 64] for i in range(8))
        k1, k2, w = (int.from_bytes(vk[640 + 32 * i:672 + 32 * i], "big") for i in range(3))
        beta = _challenge(vk[:512] + b"".join(_be(x) for x in public_inputs) + A + B + Cc)
        gamma = _challenge(_be(beta))
        alpha = _challenge(_be(beta) + _be(gamma) + Z)
        xi = _challenge(_be(alpha) + T1 + T2 + T3)
        v1 = _challenge(_be(xi) + b"".join(_be(e) for e in evs))
        v = [0, v1] + [pow(v1, i, R_MOD) for i in range(2, 6)]
        u = _challenge(Wxi + Wxiw)
        n = 1 << self.log_n
        xin = pow(xi, n, R_MOD)
        zh = (xin - 1) % R_MOD
        lag, wi = [], 1
        for _ in range(max(1, self.n_public)):
            lag.append(wi * zh * pow(n * (xi - wi), -1, R_MOD) % R_MOD)
            wi = wi * w % R_MOD
        l1 = lag[0]
        pi = -sum(x * lag[i] for i, x in enumerate(public_inputs)) % R_MOD
        a2 = alpha * alpha % R_MOD
        e3a, e3b = (ea + beta * es1 + gamma) % R_MOD, (eb + beta * es2 + gamma) % R_MOD
        r0 = (pi - l1 * a2 - alpha * e3a * e3b * (ec + gamma) * ezw) % R_MOD
        bxi = beta * xi % R_MOD
        d2a = alpha * (ea + bxi + gamma) * (eb + bxi * k1 + gamma) * (ec + bxi * k2 + gamma) % R_MOD
        d3 = alpha * beta * ezw * e3a * e3b % R_MOD
        e = (-r0 + v[1] * ea + v[2] * eb + v[3] * ec + v[4] * es1 + v[5] * es2 + u * ezw) % R_MOD
        # B1 = xi Wxi + u xi w Wxiw + D + v1 A + v2 B + v3 C + v4 S1 + v5 S2 - e [1]1 (D of calculateD), A1 = Wxi + u Wxiw
        g1 = (1).to_bytes(32, "big") + (2).to_bytes(32, "big")
        terms = [(ea * eb, Qm), (ea, Ql), (eb, Qr), (ec, Qo), (1, Qc), (d2a + l1 * a2 + u, Z), (-d3, S3), (-zh, T1), (-zh * xin, T2),
                 (-zh * xin * xin, T3), (v[1], A), (v[2], B), (v[3], Cc), (v[4], S1), (v[5], S2), (xi, Wxi), (u * xi * w, Wxiw), (-e, g1)]
        try:
            b1 = self.ctx.g1_msm(b"".join(p for _, p in terms), b"".join(_be(s) for s, _ in terms), len(terms), F.POINTS_BE | F.SCALARS_BE)
            a1 = self.ctx.g1_msm(Wxi + Wxiw, _be(1) + _be(u), 2, F.POINTS_BE | F.SCALARS_BE)
        except Exception:  # a point that is not on the curve
            return False
        y = int.from_bytes(a1[32:], "big")
        neg_a1 = a1 if y == 0 and int.from_bytes(a1[:32], "big") == 0 else a1[:32] + (P_MOD - y).to_bytes(32, "big")
        res, st = self.ctx.bn254_pairing_check_batch([neg_a1 + vk[512:640] + b1 + G2_ONE])
        return bool(res[0]) and st[0] == 0


class PlonkProver:
    """`PlonkProver(ctx, zkey, precompute=True)`: a snarkjs 0.7 PLONK .zkey (bytes or a path) loaded once;
    `prove(wtns, blinding=None)` -> the 768-byte proof of a .wtns witness in ONE call of the C ABI
    (b200zk_plonk_zkey_prove).  Blinding b1..b11 is drawn here with `random_scalar` unless given; the library draws
    none.  `precompute` builds PTau's window tables (faster MSMs, about 13x PTau's memory)."""

    def __init__(self, ctx, zkey, precompute: bool = True):
        data = _bytes(zkey)
        ptr, keep = _host_ptr(data)
        h = C.c_uint64()
        ctx._check(F.lib.b200zk_plonk_zkey_load(ctx._h, ptr, len(data), 1 if precompute else 0, C.byref(h)), "b200zk_plonk_zkey_load")
        del keep
        self.ctx, self.key = ctx, h.value
        try:
            nv, npub, log_n = C.c_uint32(), C.c_uint32(), C.c_uint32()
            vk = C.create_string_buffer(736)
            ctx._check(F.lib.b200zk_plonk_zkey_info(ctx._h, self.key, C.byref(nv), C.byref(npub), C.byref(log_n), vk, 736), "b200zk_plonk_zkey_info")
            self.n_vars, self.n_public, self.log_n = nv.value, npub.value, log_n.value
            self._vk = vk.raw
        except BaseException:
            self.close()
            raise

    def vk(self) -> bytes:
        """Qm Ql Qr Qo Qc S1 S2 S3 (64 each) | X_2 (128) | k1 | k2 | w (32 each), EIP-196/197 and big-endian"""
        return self._vk

    def verifier(self) -> PlonkVerifier:
        return PlonkVerifier(self.ctx, self._vk, self.n_public, self.log_n)

    def prove(self, wtns, blinding=None) -> bytes:
        if self.key is None:
            raise ValueError("PlonkProver is closed")
        data = _bytes(wtns)
        blinding = [random_scalar() for _ in range(11)] if blinding is None else list(blinding)
        if len(blinding) != 11 or not all(isinstance(b, int) and 0 <= b < 1 << 256 for b in blinding):
            raise ValueError("blinding must be 11 non-negative 256-bit integers")
        ptr, keep = _host_ptr(data)
        bl = C.create_string_buffer(b"".join(int(b).to_bytes(32, "little") for b in blinding), 352)
        proof = C.create_string_buffer(768)
        self.ctx._check(F.lib.b200zk_plonk_zkey_prove(self.ctx._h, self.key, ptr, len(data), bl, _current_stream_ptr(self.ctx.device), proof),
                        "b200zk_plonk_zkey_prove")
        del keep
        return proof.raw

    def close(self):
        if self.key is not None:
            self.ctx._check(F.lib.b200zk_plonk_zkey_free(self.ctx._h, self.key), "b200zk_plonk_zkey_free")
            self.key = None
