"""Big-integer reference of the EIP-4844 proof's scalar-field work -- TEST INFRASTRUCTURE ONLY (the library computes the
same on the device, bls381.cu: kzg_eval_quotient).  Blobs list p's evaluations over the 4096 roots of unity in bit-reversed
order; for a point z this returns y = p(z) and the quotient (p(X) - y) / (X - z) in the same evaluation form."""
import hashlib

import bls_ref as bls

N = bls.FIELD_ELEMENTS_PER_BLOB
_ROOTS = None


def roots_brp():
    global _ROOTS
    if _ROOTS is None:
        nat = [1] * N
        for i in range(1, N):
            nat[i] = nat[i - 1] * bls.ROOT_4096 % bls.R
        _ROOTS = [nat[bls.bit_reverse(i, 12)] for i in range(N)]
    return _ROOTS


def blob_values(blob: bytes):
    return [int.from_bytes(blob[32 * i:32 * i + 32], "big") for i in range(N)]


def to_blob(vals) -> bytes:
    return b"".join(v.to_bytes(32, "big") for v in vals)


def quotient(poly, z: int):
    """-> (q, y): q_i = (p_i - y) / (w_i - z), with the spec's special case when z = w_m (c-kzg compute_kzg_proof_impl)"""
    r, roots = bls.R, roots_brp()
    if z in roots:
        m = roots.index(z)
        y = poly[m]
        q = [0] * N
        zinv = pow(z, -1, r)
        for i, w in enumerate(roots):
            if i == m:
                continue
            q[i] = (poly[i] - y) * pow((w - z) % r, -1, r) % r
            q[m] = (q[m] + (poly[i] - y) * w % r * zinv % r * pow((z - w) % r, -1, r)) % r
        return q, y
    # barycentric evaluation: p(z) = (z^n - 1)/n * sum_i p_i w_i / (z - w_i)
    inv = [pow((z - w) % r, -1, r) for w in roots]
    acc = sum(p * w % r * d for p, w, d in zip(poly, roots, inv)) % r
    y = (pow(z, N, r) - 1) * pow(N, -1, r) % r * acc % r
    return [(y - p) * d % r for p, d in zip(poly, inv)], y


def challenge(blob: bytes, commitment: bytes) -> int:
    """EIP-4844 compute_challenge: hash_to_bls_field(domain | degree as 16-byte big-endian | blob | commitment)"""
    data = b"FSBLOBVERIFY_V1_" + N.to_bytes(16, "big") + blob + commitment
    return int.from_bytes(hashlib.sha256(data).digest(), "big") % bls.R


def evaluate_direct(poly, z: int) -> int:
    """p(z) through the Lagrange basis at z (the definition, O(n) inversions): independent of `quotient`'s formula"""
    return sum(v * l for v, l in zip(poly, bls.lagrange_setup_scalars(z))) % bls.R if z not in roots_brp() else poly[roots_brp().index(z)]
