"""EIP-4844 blob commitments on the library's CUDA kernels: the host-side mirror of the reference's `crypto::kzg` surface
(/root/reference/crates/common/crypto/kzg.rs:259-293, used by /root/reference/crates/common/types/blobs_bundle.rs:90-118
and the L2 committer, crates/l2/sequencer/l1_committer.rs:1488-1521).

    blob_to_kzg_commitment(blob)               one 4096-point BLS12-381 G1 MSM over the Lagrange-form trusted setup
    compute_kzg_proof(blob, z)                 p(z) by the barycentric formula + the quotient's commitment (a second MSM)
    compute_blob_kzg_proof(blob, commitment)   the same at the Fiat-Shamir challenge of EIP-4844
    blob_to_kzg_commitment_and_proof(blob)     what `BlobsBundle::create_from_blobs` calls per blob (wrapper version 0)

With a `Context` everything runs in libb200zk.so: the MSMs, and the scalar-field work of a proof (p(z), the quotient, its
4096 inverses as one batch) in a CUDA kernel (`b200zk_kzg_compute_proof`, `b200zk_kzg_blob_to_commitment_and_proof`); the
library hashes the challenge itself.  `compute_challenge` below is the same hash in Python, for callers that pass a
commitment in.  KzgSettings also accepts a context object that serves only the two MSM calls (`kzg_blob_to_commitment`,
`bls12_381_g1_msm_resident`); for such an object the proof's scalar-field work is done here in Python integers.  The
trusted setup is an INPUT (4096 compressed G1 points in c-kzg's g1_lagrange_brp order): the reference gets it from inside the
c-kzg / kzg-rs crates, which are not in the tree, so no setup is bundled here.

Verification (verify_kzg_proof, verify_blob_kzg_proof, verify_blob_kzg_proof_batch) needs the setup's G2 points as well
(`g2_monomial`: at least [1]2 and [tau]2, 96-byte compressed) and a `Context`: the pairing runs on the device
(`b200zk_kzg_verify_proof_batch`, `b200zk_kzg_verify_blob_proof_batch`).

EIP-7594 cells (wrapper version 1, crates/common/crypto/kzg.rs:72-113 of the reference): `compute_cells` extends a blob to
its 128 cells and `verify_cell_kzg_proof_batch` checks every cell proof of a bundle in one pairing check, both on the
device (`b200zk_kzg_compute_cells`, `b200zk_kzg_verify_cell_proof_batch`); verification needs `g2_monomial` with all 65
points ([tau^64]2 is point 64).  `blob_to_commitment_and_cell_proofs` (kzg.rs:275-293, what `BlobsBundle::create_from_blobs`
calls per blob for wrapper version 1) computes the commitment and the 128 cell proofs by FK20 on the device
(`b200zk_kzg_blob_to_commitment_and_cell_proofs`); it needs `g1_monomial`, the setup's 4096 points [tau^i]1.
"""
from __future__ import annotations

import hashlib

from .errors import B200Error

BLS_MODULUS = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001
FIELD_ELEMENTS_PER_BLOB = 4096
BYTES_PER_BLOB = 32 * FIELD_ELEMENTS_PER_BLOB
FIELD_ELEMENTS_PER_CELL = 64
CELLS_PER_EXT_BLOB = 128
BYTES_PER_CELL = 32 * FIELD_ELEMENTS_PER_CELL
FIAT_SHAMIR_PROTOCOL_DOMAIN = b"FSBLOBVERIFY_V1_"
PRIMITIVE_ROOT_OF_UNITY = 7


def _bit_reverse(i: int, bits: int) -> int:
    return int(format(i, f"0{bits}b")[::-1], 2)


_ROOTS_BRP = None


def roots_of_unity_brp():
    """the 4096 roots of unity in bit-reversed order (the order blobs list their evaluations in)"""
    global _ROOTS_BRP
    if _ROOTS_BRP is None:
        w = pow(PRIMITIVE_ROOT_OF_UNITY, (BLS_MODULUS - 1) // FIELD_ELEMENTS_PER_BLOB, BLS_MODULUS)
        nat = [1] * FIELD_ELEMENTS_PER_BLOB
        for i in range(1, FIELD_ELEMENTS_PER_BLOB):
            nat[i] = nat[i - 1] * w % BLS_MODULUS
        _ROOTS_BRP = [nat[_bit_reverse(i, 12)] for i in range(FIELD_ELEMENTS_PER_BLOB)]
    return _ROOTS_BRP


class KzgSettings:
    """The trusted setup resident in HBM (the reference's `c_kzg::ethereum_kzg_settings(KZG_PRECOMPUTE)`, kzg.rs:262)."""

    def __init__(self, ctx, g1_lagrange_brp: bytes, precompute: bool = True, g2_monomial: bytes | None = None,
                 g1_monomial: bytes | None = None):
        if len(g1_lagrange_brp) != 48 * FIELD_ELEMENTS_PER_BLOB:
            raise ValueError("the setup is 4096 compressed G1 points (48 bytes each) in g1_lagrange_brp order")
        if g2_monomial is not None and (len(g2_monomial) % 96 or len(g2_monomial) < 2 * 96):
            raise ValueError("g2_monomial is at least 2 compressed G2 points (96 bytes each): [1]2, [tau]2, ...")
        if g1_monomial is not None and len(g1_monomial) != 48 * FIELD_ELEMENTS_PER_BLOB:
            raise ValueError("g1_monomial is 4096 compressed G1 points (48 bytes each): [tau^i]1 for i < 4096")
        self.ctx = ctx
        self.g2_handle = 0
        self.g1_monomial_handle = 0
        self.handle = ctx.bls12_381_g1_bases_upload(g1_lagrange_brp, FIELD_ELEMENTS_PER_BLOB)
        if precompute:
            ctx.bases_precompute(self.handle, 0)
        if g2_monomial is not None:
            self.g2_handle = ctx.bls12_381_g2_bases_upload(g2_monomial, len(g2_monomial) // 96)
        if g1_monomial is not None:
            self.g1_monomial_handle = ctx.bls12_381_g1_bases_upload(g1_monomial, FIELD_ELEMENTS_PER_BLOB)

    def close(self):
        for name in ("handle", "g2_handle", "g1_monomial_handle"):
            if getattr(self, name):
                self.ctx.bases_free(getattr(self, name))
                setattr(self, name, 0)

    # ---- kzg.rs:259-272
    def blob_to_kzg_commitment(self, blob: bytes) -> bytes:
        if len(blob) != BYTES_PER_BLOB:
            raise ValueError("a blob is 131072 bytes")
        return self.ctx.kzg_blob_to_commitment(self.handle, blob)[0]

    def blobs_to_kzg_commitments(self, blobs) -> list:
        return self.ctx.kzg_blob_to_commitment(self.handle, b"".join(blobs)) if blobs else []

    def _one_call(self) -> bool:
        """a `Context` proves in one device call; an object that serves only the two MSM calls does not"""
        return hasattr(self.ctx, "kzg_compute_proof")

    def compute_kzg_proof(self, blob: bytes, z: int):
        """-> (proof 48 bytes, y = p(z)): p(z) by the barycentric formula and the commitment of the quotient
        (p(x) - y) / (x - z).  With a `Context` both are computed on the device (`b200zk_kzg_compute_proof`)."""
        if not 0 <= z < BLS_MODULUS:
            raise ValueError("field element out of range")
        if not self._one_call():
            return self._compose_proof(blob, z)
        try:
            proofs, ys = self.ctx.kzg_compute_proof(self.handle, blob, z.to_bytes(32, "big"))
        except B200Error as e:
            if e.status == 2:  # a blob element >= r (c-kzg: C_KZG_BADARGS)
                raise ValueError("field element out of range") from e
            raise
        return proofs[0], int.from_bytes(ys[0], "big")

    def _compose_proof(self, blob: bytes, z: int):
        """For a context object that offers only `bls12_381_g1_msm_resident` and `kzg_blob_to_commitment` (the MSM calls):
        the scalar-field work in Python integers, as c-kzg does it on the CPU, then one MSM over the quotient.  A `Context`
        never takes this path."""
        poly = [int.from_bytes(blob[32 * i:32 * i + 32], "big") for i in range(FIELD_ELEMENTS_PER_BLOB)]
        if any(v >= BLS_MODULUS for v in poly):
            raise ValueError("field element out of range")
        roots = roots_of_unity_brp()
        r = BLS_MODULUS
        if z in roots:
            m = roots.index(z)
            y = poly[m]
            # q_m = sum_{i != m} (p_i - y) w_i / (z (z - w_i));  q_i = (p_i - y) / (w_i - z) elsewhere
            q = [0] * FIELD_ELEMENTS_PER_BLOB
            zinv = pow(z, -1, r)
            for i, w in enumerate(roots):
                if i == m:
                    continue
                q[i] = (poly[i] - y) * pow((w - z) % r, -1, r) % r
                q[m] = (q[m] + (poly[i] - y) * w % r * zinv % r * pow((z - w) % r, -1, r)) % r
        else:
            # barycentric evaluation: p(z) = (z^n - 1)/n * sum_i p_i w_i / (z - w_i)
            inv = [pow((z - w) % r, -1, r) for w in roots]
            acc = sum(p * w % r * d for p, w, d in zip(poly, roots, inv)) % r
            y = (pow(z, FIELD_ELEMENTS_PER_BLOB, r) - 1) * pow(FIELD_ELEMENTS_PER_BLOB, -1, r) % r * acc % r
            q = [(y - p) * d % r for p, d in zip(poly, inv)]  # (p_i - y)/(w_i - z) = (y - p_i)/(z - w_i)
        scalars = b"".join(v.to_bytes(32, "big") for v in q)
        return self.ctx.bls12_381_g1_msm_resident(self.handle, scalars, FIELD_ELEMENTS_PER_BLOB), y

    @staticmethod
    def compute_challenge(blob: bytes, commitment: bytes) -> int:
        """EIP-4844 compute_challenge: hash_to_bls_field(domain | degree (16 B BE) | blob | commitment)"""
        data = FIAT_SHAMIR_PROTOCOL_DOMAIN + FIELD_ELEMENTS_PER_BLOB.to_bytes(16, "big") + blob + commitment
        return int.from_bytes(hashlib.sha256(data).digest(), "big") % BLS_MODULUS

    def compute_blob_kzg_proof(self, blob: bytes, commitment: bytes) -> bytes:
        return self.compute_kzg_proof(blob, self.compute_challenge(blob, commitment))[0]

    def blob_to_kzg_commitment_and_proof(self, blob: bytes):
        """the commitment and the proof at the Fiat-Shamir challenge, in one device call"""
        if not self._one_call():
            c = self.blob_to_kzg_commitment(blob)
            return c, self.compute_blob_kzg_proof(blob, c)
        if len(blob) != BYTES_PER_BLOB:
            raise ValueError("a blob is 131072 bytes")
        commitments, proofs = self.ctx.kzg_blob_to_commitment_and_proof(self.handle, blob)
        return commitments[0], proofs[0]

    def blobs_to_kzg_commitments_and_proofs(self, blobs) -> tuple:
        """([commitments], [proofs]) for a batch of blobs in one device call"""
        if not self._one_call():
            pairs = [self.blob_to_kzg_commitment_and_proof(b) for b in blobs]
            return [c for c, _ in pairs], [p for _, p in pairs]
        return self.ctx.kzg_blob_to_commitment_and_proof(self.handle, b"".join(blobs)) if blobs else ([], [])

    # ---- verification: provider.rs:463-544, kzg.rs:168-192
    def _verifier(self) -> int:
        if not hasattr(self.ctx, "kzg_verify_proof_batch"):
            raise TypeError("KZG verification runs on the device: KzgSettings needs a Context")
        if not self.g2_handle:
            raise ValueError("KZG verification needs the setup's G2 points: pass g2_monomial")
        return self.g2_handle

    def verify_kzg_proof(self, commitment: bytes, z, y, proof: bytes) -> bool:
        """c-kzg verify_kzg_proof: does `proof` open `commitment` to y at z?  z, y: ints or 32-byte big-endian.  Raises
        ValueError on malformed input (c-kzg's C_KZG_BADARGS): z or y >= r, or an invalid commitment or proof."""
        h = self._verifier()
        zb, yb = (v.to_bytes(32, "big") if isinstance(v, int) else bytes(v) for v in (z, y))
        if len(commitment) != 48 or len(proof) != 48 or len(zb) != 32 or len(yb) != 32:
            raise ValueError("commitment and proof are 48 bytes, z and y 32 bytes")
        res, st = self.ctx.kzg_verify_proof_batch(h, commitment, zb, yb, proof)
        if st[0] in (2, 3):
            raise ValueError("field element out of range" if st[0] == 2 else "invalid commitment or proof")
        return res[0] == 1

    def verify_blob_kzg_proof(self, blob: bytes, commitment: bytes, proof: bytes) -> bool:
        """c-kzg verify_blob_kzg_proof: a batch of one"""
        return self.verify_blob_kzg_proof_batch([blob], [commitment], [proof])

    def verify_blob_kzg_proof_batch(self, blobs, commitments, proofs) -> bool:
        """c-kzg verify_blob_kzg_proof_batch: one answer for the batch; ValueError on malformed input"""
        h = self._verifier()
        if not len(blobs) == len(commitments) == len(proofs):
            raise ValueError("blobs, commitments and proofs differ in length")
        if any(len(b) != BYTES_PER_BLOB for b in blobs) or any(len(c) != 48 for c in commitments) or any(len(p) != 48 for p in proofs):
            raise ValueError("a blob is 131072 bytes, a commitment and a proof 48 bytes")
        try:
            return self.ctx.kzg_verify_blob_proof_batch(h, b"".join(blobs), b"".join(commitments), b"".join(proofs))
        except B200Error as e:
            if e.status in (2, 3):
                raise ValueError(str(e)) from e
            raise

    # ---- EIP-7594 cells: kzg.rs:72-113, blobs_bundle.rs:152-173
    def compute_cells(self, blob: bytes) -> list:
        """c-kzg compute_cells: the blob's 128 cells of 2048 bytes; the first 64 are the blob itself.  ValueError when a
        blob element is >= r."""
        if not hasattr(self.ctx, "kzg_compute_cells"):
            raise TypeError("compute_cells runs on the device: KzgSettings needs a Context")
        if len(blob) != BYTES_PER_BLOB:
            raise ValueError("a blob is 131072 bytes")
        try:
            return self.ctx.kzg_compute_cells(blob)[0]
        except B200Error as e:
            if e.status == 2:
                raise ValueError(str(e)) from e
            raise

    def blob_to_commitment_and_cell_proofs(self, blob: bytes):
        """kzg::blob_to_commitment_and_cell_proofs (c-kzg compute_cells_and_kzg_proofs): (commitment, [128 cell proofs]),
        48 bytes each.  ValueError when a blob element is >= r."""
        if len(blob) != BYTES_PER_BLOB:
            raise ValueError("a blob is 131072 bytes")
        commitments, proofs = self.blobs_to_commitments_and_cell_proofs([blob])
        return commitments[0], proofs

    def blobs_to_commitments_and_cell_proofs(self, blobs) -> tuple:
        """([commitments], [cell proofs]) for a batch of blobs in one device call; the proofs blob-major, 128 per blob"""
        if not hasattr(self.ctx, "kzg_blob_to_commitment_and_cell_proofs"):
            raise TypeError("cell proofs are computed on the device: KzgSettings needs a Context")
        if not self.g1_monomial_handle:
            raise ValueError("cell proofs need the setup's monomial G1 points: pass g1_monomial")
        if any(len(b) != BYTES_PER_BLOB for b in blobs):
            raise ValueError("a blob is 131072 bytes")
        if not blobs:
            return [], []
        try:
            return self.ctx.kzg_blob_to_commitment_and_cell_proofs(self.handle, self.g1_monomial_handle, b"".join(blobs))
        except B200Error as e:
            if e.status == 2:
                raise ValueError(str(e)) from e
            raise

    def verify_cell_kzg_proof_batch(self, blobs, commitments, cell_proofs) -> bool:
        """verify_cell_kzg_proof_batch over whole blobs, as the reference calls it: every cell of every blob, each
        commitment once per blob, cell_proofs blob-major (128 per blob, cell index inner).  One answer; ValueError on
        malformed input"""
        h = self._verifier()
        if not len(blobs) == len(commitments) or len(cell_proofs) != CELLS_PER_EXT_BLOB * len(blobs):
            raise ValueError("need one commitment and 128 cell proofs per blob")
        if any(len(b) != BYTES_PER_BLOB for b in blobs) or any(len(c) != 48 for c in commitments) or any(len(p) != 48 for p in cell_proofs):
            raise ValueError("a blob is 131072 bytes, a commitment and a proof 48 bytes")
        try:
            return self.ctx.kzg_verify_cell_proof_batch(self.handle, h, b"".join(blobs), b"".join(commitments), b"".join(cell_proofs))
        except B200Error as e:
            if e.status in (2, 3):
                raise ValueError(str(e)) from e
            raise
