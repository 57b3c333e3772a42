"""TEST INFRASTRUCTURE: the ark-groth16 / gnark key layout of tests/groth16_toy.py's instance, and its blinded proof.

ToyGroth16 folds alpha and beta into the points of variable 0.  ark-groth16 and gnark keep them apart: the query
columns carry u_i, v_i only, and alpha1, beta1, beta2, delta1, delta2 sit beside them.  With the toxic waste known, the
blinded proof of ark-groth16 0.5 (create_proof_with_reduction) / gnark (groth16.Prove) is again one scalar
multiplication per element:
    a = alpha + sum z_i u_i + r delta          b = beta + sum z_i v_i + s delta
    c = (sum_{private} z_i k_i + h(tau) Z(tau)) / delta + s a + r b - r s delta
"""
from groth16_toy import N_PUBLIC, R, ToyGroth16, _g1, _g2  # noqa: F401


class ArkKey:
    """the toy's key in ark layout: columns without alpha / beta, plus the five key terms (EIP-196/197 bytes)"""

    def __init__(self, toy: ToyGroth16):
        self.toy = toy
        self.a_g1 = b"".join(_g1(toy.u[i]) for i in range(toy.m))
        self.b_g1 = b"".join(_g1(toy.v[i]) for i in range(toy.m))
        self.b_g2 = b"".join(_g2(toy.v[i]) for i in range(toy.m))
        self.l_g1, self.h_g1 = toy.l_g1, toy.h_g1
        self.alpha_g1, self.beta_g1, self.beta_g2 = _g1(toy.alpha), _g1(toy.beta), _g2(toy.beta)
        self.delta_g1, self.delta_g2 = _g1(toy.delta), _g2(toy.delta)

    def columns(self):
        return self.a_g1, self.b_g1, self.b_g2, self.l_g1, self.h_g1

    def terms(self):
        return self.alpha_g1, self.beta_g1, self.beta_g2, self.delta_g1, self.delta_g2


def zk_scalars(toy: ToyGroth16, z, r: int, s: int):
    """(a, b, c) of the blinded proof in the exponent, and the verification equation they satisfy"""
    a = (toy.alpha + sum(zi * ui for zi, ui in zip(z, toy.u)) + r * toy.delta) % R
    b = (toy.beta + sum(zi * vi for zi, vi in zip(z, toy.v)) + s * toy.delta) % R
    at = sum(zi * ui for zi, ui in zip(z, toy.u)) % R
    bt = sum(zi * vi for zi, vi in zip(z, toy.v)) % R
    ct = sum(zi * wi for zi, wi in zip(z, toy.w)) % R
    hz = (at * bt - ct) % R
    c0 = (sum(z[i] * toy.k[i] for i in range(N_PUBLIC, toy.m)) + hz) % R * pow(toy.delta, -1, R) % R
    c = (c0 + s * a + r * b - r * s * toy.delta) % R
    assert (a * b - toy.alpha * toy.beta - toy.gamma * sum(z[i] * toy.ic[i] for i in range(N_PUBLIC)) - toy.delta * c) % R == 0
    return a, b, c


def expected_zk_proof(toy: ToyGroth16, z, r: int, s: int) -> bytes:
    a, b, c = zk_scalars(toy, z, r, s)
    return _g1(a) + _g2(b) + _g1(c)
