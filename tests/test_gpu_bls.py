"""BLS12-381 G1 MSM and the EIP-4844 blob commitment path (SURVEY.md section 8f row 3) against the pure-Python oracle
oracle/bls_ref.py: compressed bytes in, compressed bytes out.  The reference's own KZG vectors
(/root/reference/crates/common/types/blobs_bundle.rs:430-485) are commitments under the mainnet trusted setup, which lives in
the c-kzg crate and not in the tree ("parity unpinned", see oracle/bls_ref.py); the setup here is synthetic -- Lagrange points
L_i(tau) * G for a known tau -- so that every commitment and proof has a closed form in the exponent."""
import numpy as np
import pytest

import bls_ref as bls

pytestmark = pytest.mark.gpu

import ethrex_b200 as eb  # noqa: E402
from ethrex_b200 import _ffi as F  # noqa: E402

TAU = 0x5A3C91E7B2D4F60819ACBD3E57F1024689BDF0135792468ACE0FDB9753102468 % bls.R


def _scalars(n, seed=1):
    rng = np.random.default_rng(seed)
    vals = [int.from_bytes(rng.bytes(32), "big") % bls.R for _ in range(n)]
    special = [0, 1, 2, bls.R - 1, bls.R - 2, 1 << 254, (1 << 128) - 1]
    for i, v in enumerate(special):
        if i < n:
            vals[(i * 7919) % n] = v % bls.R
    return vals


@pytest.mark.parametrize("n,table", [(1, False), (2, False), (33, False), (300, False), (300, True)])
def test_bls12_381_g1_msm_matches_oracle(ctx, n, table):
    ks = [(3 + 5 * i) * 0x9E3779B97F4A7C15 % bls.R for i in range(n)]
    pts = bls.generator_multiples(ks)
    if n >= 33:
        pts[7] = None            # an identity point among the bases
        pts[9] = pts[8]          # a repeated point
        pts[11] = (pts[10][0], bls.P - pts[10][1])  # P and -P
    s = _scalars(n)
    exp = bls.compress(bls.msm(s, pts))
    h = ctx.bls12_381_g1_bases_upload(b"".join(bls.compress(p) for p in pts), n)
    try:
        if table:
            ctx.bases_precompute(h, 0)
        assert ctx.bls12_381_g1_msm_resident(h, b"".join(v.to_bytes(32, "big") for v in s), n) == exp
        # little-endian limbs (range-checked like big-endian ones): same bytes
        le = b"".join(v.to_bytes(32, "little") for v in s)
        assert ctx.bls12_381_g1_msm_resident(h, le, n, 0) == exp
        # all-zero scalars: the identity, in its compressed form
        assert ctx.bls12_381_g1_msm_resident(h, bytes(32 * n), n) == bytes([0xC0]) + bytes(47)
    finally:
        ctx.bases_free(h)
    # the same points uncompressed
    h2 = ctx.bls12_381_g1_bases_upload(b"".join(bls.uncompressed(p) for p in pts), n, 0)
    try:
        assert ctx.bls12_381_g1_msm_resident(h2, b"".join(v.to_bytes(32, "big") for v in s), n) == exp
    finally:
        ctx.bases_free(h2)


def test_bls12_381_generator_roundtrip_and_group_order(ctx):
    """public constants: the compressed generator decodes, 1 * G re-encodes to the same 48 bytes, (r - 1) * G = -G"""
    h = ctx.bls12_381_g1_bases_upload(bls.G1_COMPRESSED, 1)
    try:
        assert ctx.bls12_381_g1_msm_resident(h, (1).to_bytes(32, "big"), 1) == bls.G1_COMPRESSED
        neg = bls.compress((bls.G1[0], bls.P - bls.G1[1]))
        assert ctx.bls12_381_g1_msm_resident(h, (bls.R - 1).to_bytes(32, "big"), 1) == neg
        assert ctx.bls12_381_g1_msm_resident(h, (7).to_bytes(32, "big"), 1) == bls.compress(bls.mul(7, bls.G1))
    finally:
        ctx.bases_free(h)


def test_bls12_381_input_errors(ctx):
    g = bytearray(bls.G1_COMPRESSED)
    ok = bytes(g)
    # x >= p
    big = bytearray((bls.P + 5).to_bytes(48, "big")); big[0] |= 0x80
    with pytest.raises(eb.B200Error) as e:
        ctx.bls12_381_g1_bases_upload(ok + bytes(big), 2)
    assert e.value.kind == "Serialization"
    # x with x^3 + 4 a non-residue: not a curve point
    x = 1
    while pow((x ** 3 + 4) % bls.P, (bls.P - 1) // 2, bls.P) == 1:
        x += 1
    bad = bytearray(x.to_bytes(48, "big")); bad[0] |= 0x80
    with pytest.raises(eb.B200Error):
        ctx.bls12_381_g1_bases_upload(bytes(bad), 1)
    # compression flag missing / infinity with a non-zero x / uncompressed point off the curve
    nf = bytearray(ok); nf[0] &= 0x7F
    with pytest.raises(eb.B200Error):
        ctx.bls12_381_g1_bases_upload(bytes(nf), 1)
    inf = bytearray(ok); inf[0] |= 0x40
    with pytest.raises(eb.B200Error):
        ctx.bls12_381_g1_bases_upload(bytes(inf), 1)
    off = bls.G1[0].to_bytes(48, "big") + ((bls.G1[1] + 1) % bls.P).to_bytes(48, "big")
    with pytest.raises(eb.B200Error):
        ctx.bls12_381_g1_bases_upload(off, 1, 0)
    # a scalar >= r in a big-endian call; a BLS handle in a BN254 call and vice versa
    h = ctx.bls12_381_g1_bases_upload(ok, 1)
    try:
        with pytest.raises(eb.B200Error):
            ctx.bls12_381_g1_msm_resident(h, bls.R.to_bytes(32, "big"), 1)
        with pytest.raises(eb.B200Error):
            ctx.g1_msm_resident(h, bytes(32), 1)
        with pytest.raises(eb.B200Error):
            ctx.kzg_blob_to_commitment(h, bytes(4096 * 32))  # a 1-point "setup"
    finally:
        ctx.bases_free(h)


@pytest.fixture(scope="module")
def synthetic_setup():
    lag = bls.lagrange_setup_scalars(TAU)
    return lag, bls.generator_multiples(lag)


def test_kzg_blob_commitment_and_proof_closed_form(ctx, synthetic_setup):
    """blob_to_kzg_commitment_and_proof (kzg.rs:259-272) over a synthetic Lagrange setup: the commitment must be p(tau) * G
    and the proof ((p(tau) - p(z)) / (tau - z)) * G, both computed in the exponent by the oracle."""
    from ethrex_b200.kzg import BLS_MODULUS, KzgSettings, roots_of_unity_brp
    lag, pts = synthetic_setup
    assert BLS_MODULUS == bls.R
    # spot-check the setup itself against the slow, obviously-correct scalar multiplication
    for i in (0, 1, 2047, 4095):
        assert pts[i] == bls.mul(lag[i], bls.G1)
    settings = KzgSettings(ctx, b"".join(bls.compress(p) for p in pts))
    try:
        rng = np.random.default_rng(4844)
        blobs = []
        for b in range(6):
            vals = [int.from_bytes(rng.bytes(32), "big") % bls.R for _ in range(4096)]
            if b == 1:
                vals = [0] * 4096  # the all-zero blob: the identity commitment
            if b == 2:
                vals[5], vals[6], vals[7] = bls.R - 1, 0, 1
            if b == 3:
                vals = [bls.R - 1] * 4096  # every element at the top of the field: -(sum_i L_i(tau)) = -1
            if b in (4, 5):
                vals = [0] * 4096  # one non-zero element, at the first and at the last Lagrange point
                vals[0 if b == 4 else 4095] = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF % bls.R
            blobs.append(b"".join(v.to_bytes(32, "big") for v in vals))
        commitments = settings.blobs_to_kzg_commitments(blobs)  # all six in one call
        assert len(commitments) == 6
        assert commitments[3] == bls.compress((bls.G1[0], bls.P - bls.G1[1]))  # sum_i L_i = 1, times r - 1
        for blob, c in zip(blobs, commitments):
            vals = [int.from_bytes(blob[32 * i:32 * i + 32], "big") for i in range(4096)]
            p_tau = sum(v * l for v, l in zip(vals, lag)) % bls.R
            assert c == bls.compress(bls.mul(p_tau, bls.G1))
            assert c == settings.blob_to_kzg_commitment(blob)
            c2, proof = settings.blob_to_kzg_commitment_and_proof(blob)
            assert c2 == c
            z = settings.compute_challenge(blob, c)
            proof_z, y = settings.compute_kzg_proof(blob, z)
            assert proof_z == proof
            q_tau = (p_tau - y) * pow((TAU - z) % bls.R, -1, bls.R) % bls.R
            assert proof == bls.compress(bls.mul(q_tau, bls.G1))
        # evaluation point inside the domain (the spec's special case)
        z = roots_of_unity_brp()[77]
        vals = [int.from_bytes(blobs[0][32 * i:32 * i + 32], "big") for i in range(4096)]
        proof, y = settings.compute_kzg_proof(blobs[0], z)
        assert y == vals[77]
        p_tau = sum(v * l for v, l in zip(vals, lag)) % bls.R
        assert proof == bls.compress(bls.mul((p_tau - y) * pow((TAU - z) % bls.R, -1, bls.R) % bls.R, bls.G1))
        # a field element >= r makes the blob invalid (c-kzg: C_KZG_BADARGS)
        badblob = bytearray(blobs[0]); badblob[0:32] = bls.R.to_bytes(32, "big")
        with pytest.raises(eb.B200Error):
            settings.blob_to_kzg_commitment(bytes(badblob))
    finally:
        settings.close()
