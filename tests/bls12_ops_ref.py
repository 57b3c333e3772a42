"""EIP-2537 G1/G2 addition and MSM reference -- TEST INFRASTRUCTURE ONLY (the library's are ethrex_b200/csrc/bls_ops.cu).

The group arithmetic is the independent oracles' (oracle/bls_ref.py for G1, tests/bls_pairing_ref.py for G2, both affine
chord-and-tangent); this module puts the two groups behind one interface and adds what the precompile tests need: chain
bases P_i = (a + i d) G, whose MSM has the closed form ((sum_i k_i (a + i d)) mod r) G, the MSM calldata encoding, and
the precompile's output for a list of (point, scalar) pairs."""
import bls_pairing_ref as B
import bls_ref as bls

P, R = B.P, B.R


class Group:
    def __init__(self, name, size, gen, add, neg, on_curve, in_subgroup, encode, random_point):
        self.name, self.size, self.pair = name, size, size + 32
        self.gen, self.add, self.neg, self.on_curve, self.in_subgroup = gen, add, neg, on_curve, in_subgroup
        self.encode, self.random_point = encode, random_point

    def mul(self, k, p):
        """k p for any point (no reduction of k: correct outside the subgroup too)"""
        acc = None
        while k:
            if k & 1:
                acc = self.add(acc, p)
            p = self.add(p, p)
            k >>= 1
        return acc

    def chain(self, n, a, d):
        """P_i = (a + i d) G, i < n"""
        pt, step, out = self.mul(a % R, self.gen), self.mul(d % R, self.gen), []
        for _ in range(n):
            out.append(pt)
            pt = self.add(pt, step)
        return out

    def chain_msm(self, scalars, a, d):
        """the closed form of sum_i k_i P_i over chain(len(scalars), a, d)"""
        return self.mul(sum(k * (a + i * d) for i, k in enumerate(scalars)) % R, self.gen)

    def msm(self, pairs):
        """the precompile's result for subgroup points (k P = (k mod r) P there)"""
        acc = None
        for p, k in pairs:
            acc = self.add(acc, self.mul(k % R, p))
        return acc

    def calldata(self, pairs) -> bytes:
        return b"".join(self.encode(p) + (k % (1 << 256)).to_bytes(32, "big") for p, k in pairs)


def _g1_neg(p):
    return None if p is None else (p[0], -p[1] % P)


G1 = Group("G1", 128, B.G1, bls.add, _g1_neg, bls.on_curve, B.g1_in_subgroup, B.g1_eip2537, B.g1_random_point)
G2 = Group("G2", 256, B.G2, B.g2_add, B.g2_neg, B.g2_on_curve, B.g2_in_subgroup, B.g2_eip2537, B.g2_random_point)

# (0, 2) is on E(Fp): y^2 = 0 + 4.  Points with x = 0 are the curve's inflection points, of order 3, so outside G1
G1_OFF_SUBGROUP = (0, 2)
