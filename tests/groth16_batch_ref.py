"""TEST INFRASTRUCTURE: Groth16 batch verification restated in Python (b200zk_groth16_verify_batch, include/b200zk.h).

- `SimKey` / `SimKey.proof`: valid Groth16 proofs in any number, from the known toxic waste of tests/groth16_toy.py's
  setup.  With random a, b:  A = [a]1, B = [b]2, C = [(a b - alpha beta - gamma sum_j x_j ic_j) / delta]1, where x_0 = 1
  and IC_j = [ic_j]1.  Three oracle scalar multiplications per proof, each proof with its own A, B and C.
- `batch_rhos`: the Fiat-Shamir coefficients, byte for byte as the header states them.
- `combined_pairs` / `combined_check`: the one pairing product of the batch over oracle/pyref.py's pairing, and
  `single_check`: one proof's own 4-pair check (the per-proof reference on the CPU).
- `combined_exponent`: the same combined equation in the exponent, for proofs whose discrete logs are known.
"""
import hashlib
import random

import cpu_oracle as orc
import pyref as o
from groth16_toy import ToyGroth16

R, P = o.R, o.P
TAG = b"b200zk-groth16-batch-v1"


def g1(k: int) -> bytes:
    return orc.g1_mul_be(o.g1_to_be(o.G1_GEN), (k % R).to_bytes(32, "big"))[1]


def g2(k: int) -> bytes:
    return orc.g2_mul_be(o.g2_to_be(o.G2_GEN), (k % R).to_bytes(32, "big"))[1]


_TOY = None


def toy() -> ToyGroth16:
    global _TOY
    if _TOY is None:
        _TOY = ToyGroth16(2)
    return _TOY


class SimKey:
    """a verifying key with known toxic waste: alpha, beta, gamma, delta of the toy setup, n_pub + 1 IC scalars"""

    def __init__(self, n_pub: int, seed: int = 1):
        t = toy()
        rng = random.Random(seed)
        self.n_pub = n_pub
        self.alpha, self.beta, self.gamma, self.delta = t.alpha, t.beta, t.gamma, t.delta
        self.ic = (list(t.ic) + [rng.randrange(1, R) for _ in range(n_pub + 1)])[:n_pub + 1]
        self.vk = g1(self.alpha) + g2(self.beta) + g2(self.gamma) + g2(self.delta) + b"".join(g1(k) for k in self.ic)
        self.rng = random.Random(seed ^ 0x5EED)

    def elements(self):
        """(alpha1, beta2, gamma2, delta2, [IC]) as Groth16Verifier takes them"""
        v = self.vk
        return v[:64], v[64:192], v[192:320], v[320:448], [v[448 + 64 * j: 512 + 64 * j] for j in range(self.n_pub + 1)]

    def c_scalar(self, a: int, b: int, xs) -> int:
        lin = sum(k * x for k, x in zip(self.ic, [1] + list(xs))) % R
        return (a * b - self.alpha * self.beta - self.gamma * lin) * pow(self.delta, -1, R) % R

    def proof(self, xs=None, with_logs: bool = False):
        """-> (proof bytes, public inputs) [, (a, b, c)]: a valid proof of random public inputs (or of xs)"""
        xs = [self.rng.randrange(R) for _ in range(self.n_pub)] if xs is None else list(xs)
        a, b = self.rng.randrange(1, R), self.rng.randrange(1, R)
        c = self.c_scalar(a, b, xs)
        pf = g1(a) + g2(b) + g1(c)
        return (pf, xs, (a, b, c)) if with_logs else (pf, xs)


def batch_rhos(vk: bytes, proofs, public_inputs) -> list:
    """rho_i of b200zk_groth16_verify_batch: proofs a list of 256-byte strings, public_inputs a list of lists of ints
    (each encoded as 32 bytes big-endian, as the call receives them)"""
    n = len(proofs)
    xs = b"".join(int(v).to_bytes(32, "big") for x in public_inputs for v in x)
    d = hashlib.sha256(TAG + vk + n.to_bytes(8, "big") + b"".join(proofs) + xs).digest()
    return [int.from_bytes(hashlib.sha256(d + i.to_bytes(8, "big")).digest()[:16], "big") or 1 for i in range(n)]


def proof_status(proof: bytes, xs) -> int:
    """0, 2 (a coordinate >= p or an input >= r) or 3 (A or C off the curve, B off the twist or outside the subgroup)"""
    coords = [int.from_bytes(proof[k:k + 32], "big") for k in range(0, 256, 32)]
    if any(c >= P for c in coords) or any(not 0 <= x < R for x in xs):
        return 2
    a, b, c = o.g1_from_be(proof[:64]), o.g2_from_be(proof[64:192]), o.g1_from_be(proof[192:])
    if not (o.g1_on_curve(a) and o.g1_on_curve(c) and o.g2_on_curve(b)):
        return 3
    if b is not None and o.g2_add(o.g2_mul(R - 1, b), b) is not None:  # r B != O (g2_mul reduces its scalar mod r)
        return 3
    return 0


def _vk_points(vk: bytes):
    n_ic = (len(vk) - 448) // 64
    return (o.g1_from_be(vk[:64]), o.g2_from_be(vk[64:192]), o.g2_from_be(vk[192:320]), o.g2_from_be(vk[320:448]),
            [o.g1_from_be(vk[448 + 64 * j: 512 + 64 * j]) for j in range(n_ic)])


def combined_pairs(vk: bytes, proofs, public_inputs, rhos):
    """the N + 3 pairs of the combined check over the well-formed proofs (a malformed one is left out)"""
    alpha, beta, gamma, delta, ic = _vk_points(vk)
    pairs, s, sc = [], [0] * len(ic), None
    for pf, xs, rho in zip(proofs, public_inputs, rhos):
        if proof_status(pf, xs):
            continue
        pairs.append((o.g1_mul(R - rho, o.g1_from_be(pf[:64])), o.g2_from_be(pf[64:192])))
        for j, x in enumerate([1] + list(xs)):
            s[j] = (s[j] + rho * x) % R
        sc = o.g1_add(sc, o.g1_mul(rho, o.g1_from_be(pf[192:])))
    pairs += [(o.g1_mul(s[0], alpha), beta), (o.g1_msm(s, ic), gamma), (sc, delta)]
    return pairs


def _drop_identities(pairs):
    return [(p, q) for p, q in pairs if p is not None and q is not None]


def combined_check(vk: bytes, proofs, public_inputs, rhos=None) -> bool:
    rhos = batch_rhos(vk, proofs, public_inputs) if rhos is None else rhos
    return o.pairing_check(_drop_identities(combined_pairs(vk, proofs, public_inputs, rhos)))


def single_check(vk: bytes, proof: bytes, xs) -> bool:
    """one proof's own check: e(-A, B) e(alpha, beta) e(vk_x, gamma) e(C, delta) = 1; a malformed proof is False"""
    if proof_status(proof, xs):
        return False
    alpha, beta, gamma, delta, ic = _vk_points(vk)
    vk_x = o.g1_msm([1] + list(xs), ic)
    pairs = [(o.pt_neg(o._Fq, o.g1_from_be(proof[:64])), o.g2_from_be(proof[64:192])),
             (alpha, beta), (vk_x, gamma), (o.g1_from_be(proof[192:]), delta)]
    return o.pairing_check(_drop_identities(pairs))


def combined_exponent(key: SimKey, logs, public_inputs, rhos) -> int:
    """the combined equation in the exponent (0 when it holds): sum_i rho_i (-a_i b_i + alpha beta + gamma vk_x(i) +
    delta c_i) mod r, for proofs given by their discrete logs (a_i, b_i, c_i)"""
    acc = 0
    for (a, b, c), xs, rho in zip(logs, public_inputs, rhos):
        lin = sum(k * x for k, x in zip(key.ic, [1] + list(xs)))
        acc += rho * (-a * b + key.alpha * key.beta + key.gamma * lin + key.delta * c)
    return acc % R
