"""TEST INFRASTRUCTURE: snarkjs-0.7-layout PLONK .zkey / .wtns files of a random circom-style circuit with a KNOWN tau,
a pure-Python prover that restates snarkjs 0.7's plonk_prove.js, and its verifier (plonk_verify.js).  include/b200zk.h
states the layouts; ethrex_b200/zkey.py (PlonkProver) proves them on the device.

The circuit: signal 0 is the constant 1, signals 1..n_public are public inputs, then private inputs, then gate outputs
(all in the .wtns), then the additions (ids nVars - nAdditions ..).  Rows 0..n_public-1 are the public rows
(a = the public signal, qL = 1, so that a + PI = 0 there); every other row is a random gate
    qM a b + qL a + qR b + qO c + qC = 0
whose c is a fresh gate output, with a and b drawn from earlier signals and additions.  An addition
w = f1 w[s1] + f2 w[s2] reads earlier signals and earlier additions (so chains of additions appear), and signals are
reused across rows, so the permutation has real cycles.  nConstraints is not a power of two; rows past it are zero, with
identity sigma.

The prover follows snarkjs's route for T: the unblinded numerator on the 4n roots of unity, an iFFT, divZh, plus the
blinding part Tz (snarkjs's MulZ expansion); `t_coset` computes the same T the way the device does (the blinded
polynomials on the coset 5 <w_4n>, divided by Z_H pointwise, one inverse coset transform) so that the two can be
compared.  Commitments are [p(tau)]1, exact because tau is known.
"""
import random
import struct

import numpy as np

import cpu_oracle as orc
import pyref as o
from groth16_toy import _g1, _g2
from secp256k1_ref import keccak256
from zkey_ref import R_MONT, container, le32, wtns_bytes

R, P = o.R, o.P
K1, K2 = 2, 3
COSET = 5


def mont(v: int) -> int:
    return v % R * R_MONT % R


def g1_native(k: int) -> bytes:
    """[k]1 in the zkey's native layout (Montgomery little-endian, all-zero = identity)"""
    be = _g1(k)
    x, y = int.from_bytes(be[:32], "big"), int.from_bytes(be[32:], "big")
    if x == 0 and y == 0:
        return bytes(64)
    return (x * (1 << 256) % P).to_bytes(32, "little") + (y * (1 << 256) % P).to_bytes(32, "little")


def g2_native(k: int) -> bytes:
    be = _g2(k)
    xi, xr, yi, yr = (int.from_bytes(be[i:i + 32], "big") for i in range(0, 128, 32))
    return b"".join((v * (1 << 256) % P).to_bytes(32, "little") for v in (xr, xi, yr, yi))


def fr_le(vals) -> bytes:
    return b"".join(le32(mont(v)) for v in vals)


def to_mont_array(vals) -> np.ndarray:
    """Python ints -> (len, 4) Montgomery limbs"""
    return orc.fr_to_mont(np.frombuffer(b"".join(int(v % R).to_bytes(32, "little") for v in vals), dtype=np.uint64).reshape(-1, 4).copy())


def from_mont_array(a: np.ndarray):
    b = orc.fr_from_mont(np.ascontiguousarray(a)).tobytes()
    return [int.from_bytes(b[i:i + 32], "little") for i in range(0, len(b), 32)]


def ntt(a, inverse=False, coset=None):
    """the natural-order NTT over <w_len(a)>; from 2^12 up through the C++ oracle (the fixtures at 2^16 and 2^20)"""
    if len(a) < 4096:
        return o.ntt_fast(a, inverse=inverse, coset=coset)
    log_n = len(a).bit_length() - 1
    flags = (orc.NTT_INVERSE if inverse else 0) | (orc.NTT_COSET if coset is not None else 0)
    return from_mont_array(orc.fr_ntt(to_mont_array(a), log_n, flags, coset))


def poly_eval(coef, x: int) -> int:
    acc = 0
    for c in reversed(coef):
        acc = (acc * x + c) % R
    return acc


def challenge(data: bytes) -> int:
    return int.from_bytes(keccak256(data), "big") % R


def fr_be(v: int) -> bytes:
    return (v % R).to_bytes(32, "big")


class PlonkCircuit:
    def __init__(self, n_gates: int = 9, n_public: int = 2, n_private: int = 3, n_additions: int = 5, seed: int = 0x91A4C, log_n: int | None = None,
                 chain: float = 0.5):
        rng = random.Random(seed)
        self.rng = rng
        self.n_public = n_public
        self.n_constraints = n_public + n_gates
        self.log_n = max(3, (self.n_constraints - 1).bit_length()) if log_n is None else log_n
        assert (1 << self.log_n) >= self.n_constraints
        self.n = n = 1 << self.log_n
        self.n_wtns = 1 + n_public + n_private + n_gates
        self.n_additions = n_additions
        self.n_vars = self.n_wtns + n_additions
        self.tau = rng.randrange(2, R)
        # structure: values are recomputed per witness, so keep the recipe
        self.adds = []    # (s1, s2, f1, f2)
        self.gates = []   # (qm, ql, qr, qo, qc, sa, sb, sc)
        self.order = []   # creation order: ("add", i) or ("gate", j)
        avail = list(range(1 + n_public + n_private))
        n_add_left, n_gate_left = n_additions, n_gates
        while n_add_left or n_gate_left:
            if n_add_left and (not n_gate_left or rng.random() < n_additions / (n_additions + n_gates)):
                i = len(self.adds)
                # the newest addition is read with probability `chain`, so that chains form (chain = 1: one chain)
                s1 = self.n_wtns + i - 1 if i and rng.random() < chain else rng.choice(avail)
                s2 = rng.choice(avail)
                self.adds.append((s1, s2, rng.randrange(1, R), rng.randrange(R)))
                avail.append(self.n_wtns + i)
                self.order.append(("add", i))
                n_add_left -= 1
            else:
                j = len(self.gates)
                sc = 1 + n_public + n_private + j
                self.gates.append((rng.randrange(R), rng.randrange(R), rng.randrange(R), rng.randrange(1, R), rng.randrange(R),
                                   rng.choice(avail), rng.choice(avail), sc))
                avail.append(sc)
                self.order.append(("gate", j))
                n_gate_left -= 1
        # rows: the public rows, then the gates
        self.map_a = [1 + i for i in range(n_public)] + [g[5] for g in self.gates]
        self.map_b = [0] * n_public + [g[6] for g in self.gates]
        self.map_c = [0] * n_public + [g[7] for g in self.gates]
        zero = [0] * (n - self.n_constraints)
        self.qm = [0] * n_public + [g[0] for g in self.gates] + zero
        self.ql = [1] * n_public + [g[1] for g in self.gates] + zero
        self.qr = [0] * n_public + [g[2] for g in self.gates] + zero
        self.qo = [0] * n_public + [g[3] for g in self.gates] + zero
        self.qc = [0] * n_public + [g[4] for g in self.gates] + zero
        self._sigma()
        self.q_coef = [ntt(v, inverse=True) for v in (self.qm, self.ql, self.qr, self.qo, self.qc)]
        self.s_coef = [ntt(v, inverse=True) for v in self.sigma]

    def _sigma(self):
        n, w = self.n, o.root_of_unity(self.log_n)
        wi, x = [], 1
        for _ in range(n):
            wi.append(x)
            x = x * w % R
        ids = [[v * k % R for v in wi] for k in (1, K1, K2)]
        sigma = [list(col) for col in ids]
        groups = {}
        for col, m in enumerate((self.map_a, self.map_b, self.map_c)):
            for row, s in enumerate(m):
                groups.setdefault(s, []).append((col, row))
        for pos in groups.values():
            for k, (col, row) in enumerate(pos):
                nc, nr = pos[(k + 1) % len(pos)]
                sigma[col][row] = ids[nc][nr]
        self.sigma = sigma

    # ---- witness ----
    def assign(self, public, private=None):
        """the .wtns values (signals 0 .. nVars - nAdditions - 1) for the given inputs"""
        rng = random.Random(hash(tuple(public)) & 0xffffffff)
        n_priv = self.n_wtns - 1 - self.n_public - len(self.gates)
        private = [rng.randrange(R) for _ in range(n_priv)] if private is None else private
        z = [1] + [x % R for x in public] + [x % R for x in private] + [0] * len(self.gates) + [0] * self.n_additions
        for kind, i in self.order:
            if kind == "add":
                s1, s2, f1, f2 = self.adds[i]
                z[self.n_wtns + i] = (f1 * z[s1] + f2 * z[s2]) % R
            else:
                qm, ql, qr, qo, qc, sa, sb, sc = self.gates[i]
                a, b = z[sa], z[sb]
                z[sc] = -(qm * a * b + ql * a + qr * b + qc) * pow(qo, -1, R) % R
        return z[:self.n_wtns]

    def full(self, wt):
        z = list(wt) + [0] * self.n_additions
        for i, (s1, s2, f1, f2) in enumerate(self.adds):
            z[self.n_wtns + i] = (f1 * z[s1] + f2 * z[s2]) % R
        return z

    def wire_values(self, wt):
        z = self.full(wt)
        pad = [0] * (self.n - self.n_constraints)
        return [[z[s] for s in m] + pad for m in (self.map_a, self.map_b, self.map_c)]

    # ---- files ----
    def lagrange_coef(self, i):
        e = [0] * self.n
        e[i] = 1
        return ntt(e, inverse=True)

    def ext(self, coef):
        """coefficients | evaluations on the 4n roots of unity (a zkey polynomial section)"""
        if self.n < 1024:
            return fr_le(coef) + fr_le(ntt(list(coef) + [0] * (3 * self.n)))
        m = to_mont_array(list(coef) + [0] * (3 * self.n))
        return m[:self.n].tobytes() + orc.fr_ntt(m, self.log_n + 2).tobytes()

    def commit(self, coef) -> bytes:
        return _g1(poly_eval(coef, self.tau))

    def ptau(self, ctx=None) -> bytes:
        """[tau^i]1 for i < n + 6, native; with a device context the scalar multiplications run there
        (b200zk_bn254_g1_mul_batch)"""
        n = self.n
        if ctx is None:
            return b"".join(g1_native(pow(self.tau, i, R)) for i in range(n + 6))
        powers, x = [], 1
        for _ in range(n + 6):
            powers.append(x)
            x = x * self.tau % R
        out, st = ctx.bn254_g1_mul_batch(o.g1_to_be(o.G1_GEN) * (n + 6), b"".join(v.to_bytes(32, "big") for v in powers))
        assert not any(st)
        be = np.frombuffer(out, dtype=">u8").reshape(-1, 4)[:, ::-1].astype(np.uint64)  # 32-byte big-endian words -> limbs
        return orc.fq_to_mont(np.ascontiguousarray(be)).tobytes()

    def sections(self, ctx=None):
        n = self.n
        hdr = struct.pack("<I", 32) + P.to_bytes(32, "little") + struct.pack("<I", 32) + R.to_bytes(32, "little")
        hdr += struct.pack("<IIIII", self.n_vars, self.n_public, n, self.n_additions, self.n_constraints)
        hdr += le32(mont(K1)) + le32(mont(K2))
        for c in self.q_coef + self.s_coef:
            hdr += g1_native(poly_eval(c, self.tau))
        hdr += g2_native(self.tau)
        assert len(hdr) == 796
        adds = b"".join(struct.pack("<II", s1, s2) + le32(mont(f1)) + le32(mont(f2)) for s1, s2, f1, f2 in self.adds)
        u32s = lambda m: b"".join(struct.pack("<I", s) for s in m)
        ptau = self.ptau(ctx)
        return [(1, struct.pack("<I", 2)), (2, hdr), (3, adds), (4, u32s(self.map_a)), (5, u32s(self.map_b)), (6, u32s(self.map_c))] + \
               [(7 + k, self.ext(self.q_coef[k])) for k in range(5)] + \
               [(12, b"".join(self.ext(c) for c in self.s_coef)),
                (13, b"".join(self.ext(self.lagrange_coef(i)) for i in range(max(1, self.n_public)))),
                (14, ptau), (15, b"unknown sections are skipped")]

    def zkey(self, ctx=None) -> bytes:
        return container(b"zkey", 1, self.sections(ctx))

    def wtns(self, wt) -> bytes:
        return wtns_bytes(wt)

    def vk(self) -> bytes:
        """b200zk_plonk_zkey_info's 736 bytes"""
        w = o.root_of_unity(self.log_n)
        return b"".join(self.commit(c) for c in self.q_coef + self.s_coef) + _g2(self.tau) + fr_be(K1) + fr_be(K2) + fr_be(w)

    def public(self, wt):
        z = self.full(wt)
        return [z[s] for s in self.map_a[:self.n_public]]

    # ---- the prover (snarkjs 0.7 plonk_prove.js) ----
    def prove(self, wt, blinding=None, route="root"):
        """-> (proof bytes, dict of intermediate values).  blinding = [b1..b11] (None = all zero)."""
        b = [0] + (list(blinding) if blinding is not None else [0] * 11)
        n, log_n = self.n, self.log_n
        w = o.root_of_unity(log_n)
        av, bv, cv = self.wire_values(wt)
        # round 1
        def blind(evals, factors):  # snarkjs blindCoefficients: factors[i] (X^(n+i) - X^i)
            coef = ntt(evals, inverse=True) + [0] * len(factors)
            for i, f in enumerate(factors):
                coef[n + i] = (coef[n + i] + f) % R
                coef[i] = (coef[i] - f) % R
            return coef
        A, B, Cp = blind(av, [b[2], b[1]]), blind(bv, [b[4], b[3]]), blind(cv, [b[6], b[5]])
        cm = {"A": self.commit(A), "B": self.commit(B), "C": self.commit(Cp)}
        vk = b"".join(self.commit(c) for c in self.q_coef + self.s_coef)
        beta = challenge(vk + b"".join(fr_be(av[i]) for i in range(self.n_public)) + cm["A"] + cm["B"] + cm["C"])
        gamma = challenge(fr_be(beta))
        # round 2
        s1, s2, s3 = self.sigma
        num, den, zv = 1, 1, [1]
        x = 1
        for i in range(n):
            num = num * (av[i] + beta * x + gamma) * (bv[i] + beta * K1 * x + gamma) * (cv[i] + beta * K2 * x + gamma) % R
            den = den * (av[i] + beta * s1[i] + gamma) * (bv[i] + beta * s2[i] + gamma) * (cv[i] + beta * s3[i] + gamma) % R
            zv.append(num * pow(den, -1, R) % R)
            x = x * w % R
        if zv[n] != 1:
            raise ValueError("witness does not satisfy the copy constraints")
        Z = blind(zv[:n], [b[9], b[8], b[7]])
        cm["Z"] = self.commit(Z)
        alpha = challenge(fr_be(beta) + fr_be(gamma) + cm["Z"])
        # round 3
        pi_ev = [(-av[i]) % R if i < self.n_public else 0 for i in range(n)]
        pi_coef = ntt(pi_ev, inverse=True)
        ch = dict(beta=beta, gamma=gamma, alpha=alpha)
        T = self.t_root(av, bv, cv, zv[:n], pi_coef, b, ch) if route == "root" else \
            self.t_coset(A, B, Cp, Z, pi_coef, ch)
        if any(T[3 * n + 6:]):
            raise ValueError("witness does not satisfy the gates")
        T1 = T[:n] + [b[10]]
        T2 = T[n:2 * n] + [b[11]]
        T2[0] = (T2[0] - b[10]) % R
        T3 = T[2 * n:3 * n + 6]
        T3[0] = (T3[0] - b[11]) % R
        cm["T1"], cm["T2"], cm["T3"] = self.commit(T1), self.commit(T2), self.commit(T3)
        xi = challenge(fr_be(alpha) + cm["T1"] + cm["T2"] + cm["T3"])
        # round 4
        ev = dict(a=poly_eval(A, xi), b=poly_eval(B, xi), c=poly_eval(Cp, xi), s1=poly_eval(self.s_coef[0], xi),
                  s2=poly_eval(self.s_coef[1], xi), zw=poly_eval(Z, xi * w % R))
        v1 = challenge(fr_be(xi) + b"".join(fr_be(ev[k]) for k in ("a", "b", "c", "s1", "s2", "zw")))
        v = [0, v1] + [pow(v1, i, R) for i in range(2, 6)]
        # round 5: R (snarkjs 0.7, r0 folded in), then Wxi and Wxiw
        xin = pow(xi, n, R)
        zh = (xin - 1) % R
        l1 = zh * pow(n * (xi - 1), -1, R) % R
        pi_xi = poly_eval(pi_coef, xi)
        a2 = alpha * alpha % R
        e3a = (ev["a"] + beta * ev["s1"] + gamma) % R
        e3b = (ev["b"] + beta * ev["s2"] + gamma) % R
        r0 = (pi_xi - l1 * a2 - alpha * e3a * e3b * (ev["c"] + gamma) * ev["zw"]) % R
        d2a = alpha * (ev["a"] + beta * xi + gamma) * (ev["b"] + beta * K1 * xi + gamma) * (ev["c"] + beta * K2 * xi + gamma) % R
        d3 = alpha * beta * ev["zw"] * e3a * e3b % R
        m = n + 6
        get = lambda p, i: p[i] if i < len(p) else 0
        Rp = []
        for i in range(m):
            r = (ev["a"] * ev["b"] * get(self.q_coef[0], i) + ev["a"] * get(self.q_coef[1], i) + ev["b"] * get(self.q_coef[2], i)
                 + ev["c"] * get(self.q_coef[3], i) + get(self.q_coef[4], i) + (d2a + l1 * a2) * get(Z, i) - d3 * get(self.s_coef[2], i)
                 - zh * (get(T1, i) + xin * get(T2, i) + xin * xin % R * get(T3, i))) % R
            Rp.append(r)
        Rp[0] = (Rp[0] + r0) % R
        assert poly_eval(Rp, xi) == 0
        num_xi = [(Rp[i] + v[1] * get(A, i) + v[2] * get(B, i) + v[3] * get(Cp, i) + v[4] * get(self.s_coef[0], i) + v[5] * get(self.s_coef[1], i)) % R for i in range(m)]
        num_xi[0] = (num_xi[0] - v[1] * ev["a"] - v[2] * ev["b"] - v[3] * ev["c"] - v[4] * ev["s1"] - v[5] * ev["s2"]) % R
        num_xiw = list(Z)
        num_xiw[0] = (num_xiw[0] - ev["zw"]) % R
        Wxi, Wxiw = divide_linear(num_xi, xi), divide_linear(num_xiw, xi * w % R)
        cm["Wxi"], cm["Wxiw"] = self.commit(Wxi), self.commit(Wxiw)
        proof = b"".join(cm[k] for k in ("A", "B", "C", "Z", "T1", "T2", "T3", "Wxi", "Wxiw")) + \
            b"".join(fr_be(ev[k]) for k in ("a", "b", "c", "s1", "s2", "zw"))
        return proof, dict(T=T, beta=beta, gamma=gamma, alpha=alpha, xi=xi, v1=v1)

    def t_root(self, av, bv, cv, zv, pi_coef, b, ch):
        """snarkjs 0.7 computeT: unblinded values on the 4n roots (T), the blinding part (Tz, MulZ), divZh"""
        n, n4 = self.n, 4 * self.n
        w4 = o.root_of_unity(self.log_n + 2)
        ext = lambda coef: ntt(list(coef) + [0] * (n4 - len(coef)))
        A, B, Cc, Z = (ext(ntt(v, inverse=True)) for v in (av, bv, cv, zv))
        Q = [ext(c) for c in self.q_coef]
        S = [ext(c) for c in self.s_coef]
        L1 = ext(self.lagrange_coef(0))
        PI = ext(pi_coef)
        beta, gamma, alpha = ch["beta"], ch["gamma"], ch["alpha"]
        t, tz = [], []
        x = 1
        for i in range(n4):
            zh = (pow(x, n, R) - 1) % R  # the 4 values of snarkjs's Z1 table
            ap, bp, cp = (b[2] + b[1] * x) % R, (b[4] + b[3] * x) % R, (b[6] + b[5] * x) % R
            xw = x * o.root_of_unity(self.log_n) % R
            zp = (b[7] * x * x + b[8] * x + b[9]) % R
            zwp = (b[7] * xw * xw + b[8] * xw + b[9]) % R
            a, bb, c, z, zw = A[i], B[i], Cc[i], Z[i], Z[(i + 4) % n4]
            qm, ql, qr, qo, qc = (q[i] for q in Q)
            s1, s2, s3 = (s[i] for s in S)
            e1, e1z = mul_z([a, bb], [ap, bp], zh)
            e1, e1z = e1 * qm + a * ql + bb * qr + c * qo + PI[i] + qc, e1z * qm + ap * ql + bp * qr + cp * qo
            bx = beta * x
            e2, e2z = mul_z([a + bx + gamma, bb + bx * K1 + gamma, c + bx * K2 + gamma, z], [ap, bp, cp, zp], zh)
            e3, e3z = mul_z([a + beta * s1 + gamma, bb + beta * s2 + gamma, c + beta * s3 + gamma, zw], [ap, bp, cp, zwp], zh)
            e4, e4z = (z - 1) * L1[i] * alpha * alpha, zp * L1[i] * alpha * alpha
            t.append((e1 + alpha * (e2 - e3) + e4) % R)
            tz.append((e1z + alpha * (e2z - e3z) + e4z) % R)
            x = x * w4 % R
        T = div_zh(ntt(t, inverse=True), n)
        Tz = ntt(tz, inverse=True)
        return [(u + v) % R for u, v in zip(T, Tz)]

    def t_coset(self, A, B, Cc, Z, pi_coef, ch):
        """the device's route: blinded polynomials on the coset 5 <w_4n>, N / Z_H pointwise, one inverse coset transform"""
        n, n4 = self.n, 4 * self.n
        w4 = o.root_of_unity(self.log_n + 2)
        ext = lambda coef: ntt(list(coef) + [0] * (n4 - len(coef)), coset=COSET)
        Ae, Be, Ce, Ze, PIe = (ext(p) for p in (A, B, Cc, Z, pi_coef))
        Q = [ext(c) for c in self.q_coef]
        S = [ext(c) for c in self.s_coef]
        L1 = ext(self.lagrange_coef(0))
        beta, gamma, alpha = ch["beta"], ch["gamma"], ch["alpha"]
        t = []
        x = COSET
        for i in range(n4):
            a, bb, c, z, zw = Ae[i], Be[i], Ce[i], Ze[i], Ze[(i + 4) % n4]
            qm, ql, qr, qo, qc = (q[i] for q in Q)
            bx = beta * x
            num = (a * bb * qm + a * ql + bb * qr + c * qo + PIe[i] + qc
                   + alpha * ((a + bx + gamma) * (bb + bx * K1 + gamma) * (c + bx * K2 + gamma) * z
                              - (a + beta * S[0][i] + gamma) * (bb + beta * S[1][i] + gamma) * (c + beta * S[2][i] + gamma) * zw)
                   + alpha * alpha * (z - 1) * L1[i]) % R
            t.append(num * pow((pow(x, n, R) - 1) % R, -1, R) % R)
            x = x * w4 % R
        return ntt(t, inverse=True, coset=COSET)

    # ---- the verifier (snarkjs 0.7 plonk_verify.js) ----
    def verify(self, proof: bytes, public, tau: int | None = None) -> bool:
        """snarkjs 0.7's checks.  With tau (the trapdoor) the final pairing e(-A1, [tau]2) e(B1, [1]2) = 1 is checked as
        the equivalent B1 = tau A1 in G1; without it, through the Python pairing."""
        vk = self.vk()
        return plonk_verify(vk, self.n_public, self.log_n, proof, public, tau)


def mul_z(xs, xps, zh):
    """snarkjs MulZ: prod (x_k + Z_H x'_k) = r + Z_H rz; returns (r, rz)"""
    r, full = 1, 1
    for x_, xp in zip(xs, xps):
        r = r * x_ % R
        full = full * (x_ + zh * xp) % R
    if zh == 0:  # on the roots of H: rz is the linear term of the expansion
        rz = 0
        for k in range(len(xs)):
            term = xps[k]
            for j in range(len(xs)):
                if j != k:
                    term = term * xs[j] % R
            rz = (rz + term) % R
        return r, rz
    return r, (full - r) * pow(zh, -1, R) % R


def div_zh(coef, n):
    """snarkjs Polynomial.divZh(n, 4)"""
    q = list(coef)
    for i in range(n):
        q[i] = (-q[i]) % R
    for i in range(n, 4 * n):
        q[i] = (q[i - n] - q[i]) % R
    return q


def divide_linear(coef, x0):
    """(p(X) - p(x0)) / (X - x0): q_j = sum_{i > j} c_i x0^(i - j - 1)"""
    m = len(coef)
    q = [0] * m
    for j in range(m - 2, -1, -1):
        q[j] = (coef[j + 1] + x0 * q[j + 1]) % R
    assert (coef[0] + x0 * q[0]) % R == 0, "not divisible"
    return q


def _pt(be):
    return o.g1_from_be(be)


def plonk_verify(vk: bytes, n_public: int, log_n: int, proof: bytes, public, tau: int | None = None) -> bool:
    if len(proof) != 768 or len(public) != n_public:
        return False
    pts = [proof[64 * i:64 * i + 64] for i in range(9)]
    evs = [int.from_bytes(proof[576 + 32 * i:608 + 32 * i], "big") for i in range(6)]
    for p in pts:
        x, y = int.from_bytes(p[:32], "big"), int.from_bytes(p[32:], "big")
        if x >= P or y >= P or not o.g1_on_curve(_pt(p)):
            return False
    if any(e >= R for e in evs) or any(not (0 <= x < R) for x in public):
        return False
    A, B, C, Z, T1, T2, T3, Wxi, Wxiw = pts
    ea, eb, ec, es1, es2, ezw = evs
    Qm, Ql, Qr, Qo, Qc, S1, S2, S3 = (vk[64 * i:64 * i + 64] for i in range(8))
    k1, k2, w = (int.from_bytes(vk[640 + 32 * i:672 + 32 * i], "big") for i in range(3))
    beta = challenge(vk[:512] + b"".join(fr_be(x) for x in public) + A + B + C)
    gamma = challenge(fr_be(beta))
    alpha = challenge(fr_be(beta) + fr_be(gamma) + Z)
    xi = challenge(fr_be(alpha) + T1 + T2 + T3)
    v1 = challenge(fr_be(xi) + b"".join(fr_be(e) for e in evs))
    v = [0, v1] + [pow(v1, i, R) for i in range(2, 6)]
    u = challenge(Wxi + Wxiw)
    n = 1 << log_n
    xin = pow(xi, n, R)
    zh = (xin - 1) % R
    L, wi = [], 1
    for i in range(max(1, n_public)):
        L.append(wi * zh * pow(n * (xi - wi), -1, R) % R)
        wi = wi * w % R
    l1 = L[0]
    pi = -sum(x * L[i] for i, x in enumerate(public)) % R
    a2 = alpha * alpha % R
    e3a, e3b = (ea + beta * es1 + gamma) % R, (eb + beta * es2 + gamma) % R
    r0 = (pi - l1 * a2 - alpha * e3a * e3b * (ec + gamma) * ezw) % R
    bxi = beta * xi % R
    d2a = alpha * (ea + bxi + gamma) * (eb + bxi * k1 + gamma) * (ec + bxi * k2 + gamma) % R
    d3 = alpha * beta * ezw * e3a * e3b % R
    e = (-r0 + v[1] * ea + v[2] * eb + v[3] * ec + v[4] * es1 + v[5] * es2 + u * ezw) % R
    # B1 = xi Wxi + u xi w Wxiw + D + v1 A + v2 B + v3 C + v4 S1 + v5 S2 - e G1, A1 = Wxi + u Wxiw
    terms = [(ea * eb, Qm), (ea, Ql), (eb, Qr), (ec, Qo), (1, Qc), (d2a + l1 * a2 + u, Z), (-d3, S3),
             (-zh, T1), (-zh * xin, T2), (-zh * xin * xin, T3), (v[1], A), (v[2], B), (v[3], C), (v[4], S1), (v[5], S2),
             (xi, Wxi), (u * xi * w, Wxiw)]
    b1 = o.g1_mul(-e, o.G1_GEN)
    for s, p in terms:
        b1 = o.g1_add(b1, o.g1_mul(s % R, _pt(p)))
    a1 = o.g1_add(_pt(Wxi), o.g1_mul(u, _pt(Wxiw)))
    if tau is not None:
        return o.g1_mul(tau, a1) == b1
    x2 = o.g2_from_be(vk[512:640])
    return o.pairing_check([(o.pt_neg(o._Fq, a1), x2), (b1, o.G2_GEN)])
