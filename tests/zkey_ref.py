"""TEST INFRASTRUCTURE: snarkjs-layout .zkey / .wtns files of a random circom-style R1CS with KNOWN toxic waste, and the
proof they must give, computed in the exponent (include/b200zk.h states the layouts, ethrex_b200/zkey.py proves them).

The circuit: signal 0 is the constant 1, signals 1..n_public are free public inputs, and constraint j defines the fresh
private signal 1 + n_public + j as the product of two random linear combinations of earlier signals (C row j = that
signal).  The last few fresh signals feed no later row, so they appear in no A or B row and their A, B1, B2 points are
the identity.  snarkjs adds the rows A[n_constraints + i][i] = 1 (i = 0..n_public) before it picks the domain, so the
domain is the power of two >= n_constraints + n_public + 1; n_constraints is chosen so that it is not a power of two.

Key, with u_i, v_i, w_i the QAP polynomials of signal i at tau (Lagrange basis of the domain <w_n>):
    A_i = [u_i]1  B1_i = [v_i]1  B2_i = [v_i]2  IC_i = [(beta u_i + alpha v_i + w_i) / gamma]1 (i <= n_public)
    C_i = [(beta u_i + alpha v_i + w_i) / delta]1 (i > n_public)   H_i = [L_{2i+1}(tau) / delta]1 over the doubled domain
Proof (snarkjs groth16_prove.js / rapidsnark):  a = alpha + sum w_i u_i + r delta,  b = beta + sum w_i v_i + s delta,
    c = (sum_{i > n_public} w_i k_i + h(tau) Z(tau)) / delta + s a + r b - r s delta
The H term is derived twice and the two must agree: sum_j P_j L_{2j+1}(tau), with P = a b - c on the odd coset
w_2n <w_n> from Python NTTs, and h(tau) Z(tau) = a(tau) b(tau) - c(tau).
"""
import random
import struct

import cpu_oracle as orc
import pyref as o

from groth16_toy import _g1, _g2

R, P = o.R, o.P
R_MONT = (1 << 256) % R  # Montgomery radix mod r


# ---- small field helpers ------------------------------------------------------------------------------------------------
def lagrange_at(tau: int, log_n: int):
    """[L_j(tau)] for the Lagrange basis of <w_n>, n = 2^log_n"""
    n = 1 << log_n
    w = o.root_of_unity(log_n)
    zt = (pow(tau, n, R) - 1) % R
    ninv = pow(n, -1, R)
    out, wj = [], 1
    for _ in range(n):
        out.append(zt * ninv % R * wj % R * pow((tau - wj) % R, -1, R) % R)
        wj = wj * w % R
    return out


def dft(vals, log_n: int, inverse=False):
    """natural-order DFT over <w_n> (inverse scaled by 1/n), O(n^2): the oracle's NTT"""
    n = 1 << log_n
    w = o.root_of_unity(log_n)
    if inverse:
        w = pow(w, -1, R)
    out = []
    for k in range(n):
        wk, acc, x = pow(w, k, R), 0, 1
        for v in vals:
            acc = (acc + v * x) % R
            x = x * wk % R
        out.append(acc)
    if inverse:
        ninv = pow(n, -1, R)
        out = [v * ninv % R for v in out]
    return out


# ---- encodings ----------------------------------------------------------------------------------------------------------
def le32(v: int) -> bytes:
    return int(v).to_bytes(32, "little")


def g1_native(k: int) -> bytes:
    """[k]1 as the zkey stores it: x | y Montgomery little-endian, all-zero = identity"""
    return orc.g1_be_to_native(_g1(k)).tobytes()


def g2_native(k: int) -> bytes:
    return orc.g2_be_to_native(_g2(k)).tobytes()


def container(magic: bytes, version: int, sections) -> bytes:
    """binfileutils: magic | u32 version | u32 nSections | (u32 id | u64 size | bytes)*"""
    out = magic + struct.pack("<II", version, len(sections))
    for sid, payload in sections:
        out += struct.pack("<IQ", sid, len(payload)) + payload
    return out


def coef_record(matrix: int, constraint: int, signal: int, coef: int) -> bytes:
    """one section-4 record: the value as coef * R^2 mod r (snarkjs zkey_new.js)"""
    return struct.pack("<III", matrix, constraint, signal) + le32(coef % R * R_MONT % R * R_MONT % R)


def wtns_bytes(values, prime: int = R, n8: int = 32) -> bytes:
    return container(b"wtns", 2, [(1, struct.pack("<I", n8) + prime.to_bytes(n8, "little") + struct.pack("<I", len(values))),
                                  (2, b"".join(le32(v) for v in values))])


class ZkeyCircuit:
    def __init__(self, n_constraints: int = 11, n_public: int = 2, seed: int = 0x2CE7, terms: int = 3):
        rng = random.Random(seed)
        self.rng = rng
        self.n_public, self.n_constraints = n_public, n_constraints
        self.n_vars = 1 + n_public + n_constraints
        rows = n_constraints + n_public + 1
        self.log_n = max(1, (rows - 1).bit_length())
        self.n = 1 << self.log_n
        # constraint rows (signal -> coefficient); fresh signals of the last 3 constraints feed no later row
        self.A, self.B, self.C = [], [], []
        for j in range(n_constraints):
            avail = 1 + n_public + min(j, n_constraints - 3)
            self.A.append({rng.randrange(avail): rng.randrange(1, R) for _ in range(terms)})
            self.B.append({rng.randrange(avail): rng.randrange(1, R) for _ in range(terms)})
            self.C.append({1 + n_public + j: 1})
        for i in range(n_public + 1):  # snarkjs's padding rows: the public signals (and 1) in A only
            self.A.append({i: 1}); self.B.append({}); self.C.append({})
        self.tau, self.alpha, self.beta, self.gamma, self.delta = (rng.randrange(2, R) for _ in range(5))
        lag = lagrange_at(self.tau, self.log_n)
        self.u, self.v, self.w = [0] * self.n_vars, [0] * self.n_vars, [0] * self.n_vars
        for j in range(len(self.A)):
            for i, cf in self.A[j].items(): self.u[i] = (self.u[i] + cf * lag[j]) % R
            for i, cf in self.B[j].items(): self.v[i] = (self.v[i] + cf * lag[j]) % R
            for i, cf in self.C[j].items(): self.w[i] = (self.w[i] + cf * lag[j]) % R
        self.k = [(self.beta * self.u[i] + self.alpha * self.v[i] + self.w[i]) % R for i in range(self.n_vars)]
        self.lag = lag
        self.lag2 = lagrange_at(self.tau, self.log_n + 1)

    # ---- witness ----
    def assign(self, public):
        """the satisfying assignment for the given public inputs"""
        assert len(public) == self.n_public
        z = [1] + [x % R for x in public]
        for j in range(self.n_constraints):
            left = sum(cf * z[i] for i, cf in self.A[j].items()) % R
            right = sum(cf * z[i] for i, cf in self.B[j].items()) % R
            z.append(left * right % R)
        return z

    def evaluations(self, z):
        """(A z), (B z) on the domain (zero past the last row) and c = a o b"""
        a = [sum(cf * z[i] for i, cf in row.items()) % R for row in self.A] + [0] * (self.n - len(self.A))
        b = [sum(cf * z[i] for i, cf in row.items()) % R for row in self.B] + [0] * (self.n - len(self.B))
        return a, b, [x * y % R for x, y in zip(a, b)]

    # ---- files ----
    def records(self):
        recs = [(0, j, i, cf) for j, row in enumerate(self.A) for i, cf in row.items()]
        recs += [(1, j, i, cf) for j, row in enumerate(self.B) for i, cf in row.items()]
        self.rng.shuffle(recs)
        return recs

    def sections(self, records=None):
        """the zkey's sections as (id, payload) in snarkjs's order; tests reorder and corrupt them"""
        recs = self.records() if records is None else records
        dinv, ginv = pow(self.delta, -1, R), pow(self.gamma, -1, R)
        hdr = struct.pack("<I", 32) + P.to_bytes(32, "little") + struct.pack("<I", 32) + R.to_bytes(32, "little")
        hdr += struct.pack("<III", self.n_vars, self.n_public, self.n)
        hdr += g1_native(self.alpha) + g1_native(self.beta) + g2_native(self.beta) + g2_native(self.gamma) + g1_native(self.delta) + g2_native(self.delta)
        assert len(hdr) == 660
        np1 = self.n_public + 1
        return [(1, struct.pack("<I", 1)), (2, hdr),
                (3, b"".join(g1_native(self.k[i] * ginv) for i in range(np1))),
                (4, struct.pack("<I", len(recs)) + b"".join(coef_record(*r) for r in recs)),
                (5, b"".join(g1_native(x) for x in self.u)), (6, b"".join(g1_native(x) for x in self.v)),
                (7, b"".join(g2_native(x) for x in self.v)),
                (8, b"".join(g1_native(self.k[i] * dinv) for i in range(np1, self.n_vars))),
                (9, b"".join(g1_native(self.lag2[2 * i + 1] * dinv) for i in range(self.n))),
                (10, b"contributions are skipped")]

    def zkey(self) -> bytes:
        return container(b"zkey", 1, self.sections())

    def wtns(self, z) -> bytes:
        return wtns_bytes(z)

    # ---- the proof in the exponent ----
    def h_terms(self, z):
        """h(tau) Z(tau) two ways: sum_j P_j L_{2j+1}(tau) (P on the odd coset by NTTs) and a(tau) b(tau) - c(tau)"""
        a, b, c = self.evaluations(z)
        w2n = o.root_of_unity(self.log_n + 1)
        odd = []
        for vals in (a, b, c):
            coeffs = dft(vals, self.log_n, inverse=True)
            shifted = [cf * pow(w2n, j, R) % R for j, cf in enumerate(coeffs)]
            odd.append(dft(shifted, self.log_n))
        p_odd = [(x * y - w) % R for x, y, w in zip(*odd)]
        via_coset = sum(pj * self.lag2[2 * j + 1] for j, pj in enumerate(p_odd)) % R
        at = sum(x * l for x, l in zip(a, self.lag)) % R
        bt = sum(x * l for x, l in zip(b, self.lag)) % R
        ct = sum(x * l for x, l in zip(c, self.lag)) % R
        return via_coset, (at * bt - ct) % R

    def proof_scalars(self, z, r: int, s: int):
        h_coset, h_direct = self.h_terms(z)
        assert h_coset == h_direct
        at = sum(zi * ui for zi, ui in zip(z, self.u)) % R
        bt = sum(zi * vi for zi, vi in zip(z, self.v)) % R
        a = (self.alpha + at + r * self.delta) % R
        b = (self.beta + bt + s * self.delta) % R
        c0 = (sum(z[i] * self.k[i] for i in range(self.n_public + 1, self.n_vars)) + h_coset) % R * pow(self.delta, -1, R) % R
        c = (c0 + s * a + r * b - r * s * self.delta) % R
        return a, b, c

    def expected_proof(self, z, r: int = 0, s: int = 0) -> bytes:
        a, b, c = self.proof_scalars(z, r, s)
        return _g1(a) + _g2(b) + _g1(c)

    def verifies(self, z, r: int, s: int) -> bool:
        """the Groth16 verification equation in the exponent"""
        a, b, c = self.proof_scalars(z, r, s)
        ic = sum(z[i] * self.k[i] for i in range(self.n_public + 1)) * pow(self.gamma, -1, R) % R
        return (a * b - self.alpha * self.beta - self.gamma * ic - self.delta * c) % R == 0

    def vk(self) -> bytes:
        """alpha1 | beta2 | gamma2 | delta2 | IC as EIP-196/197 bytes (b200zk_groth16_zkey_info)"""
        ginv = pow(self.gamma, -1, R)
        return _g1(self.alpha) + _g2(self.beta) + _g2(self.gamma) + _g2(self.delta) + b"".join(_g1(self.k[i] * ginv) for i in range(self.n_public + 1))
