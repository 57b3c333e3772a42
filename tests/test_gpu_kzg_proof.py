"""EIP-4844 proofs on the device (b200zk_kzg_blob_to_commitment_and_proof, b200zk_kzg_compute_proof) over a synthetic
Lagrange setup with known tau: every commitment must be [p(tau)]G and every proof [(p(tau) - y) / (tau - z)]G, computed in
the exponent by the oracle; y must equal the big-integer reference (tests/kzg_ref.py).  Plain bases and a window table."""
import ctypes as C

import numpy as np
import pytest

import bls_ref as bls
import kzg_ref as ref

pytestmark = pytest.mark.gpu

import ethrex_b200 as eb  # noqa: E402
from ethrex_b200 import _ffi as F  # noqa: E402

TAU = 0x2F1B7C93D4A5E6F708192A3B4C5D6E7F8091A2B3C4D5E6F708192A3B4C5D6E7F % bls.R
SPECIAL = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF % bls.R


@pytest.fixture(scope="module")
def lag():
    return bls.lagrange_setup_scalars(TAU)


@pytest.fixture(scope="module")
def points(lag):
    return b"".join(bls.compress(p) for p in bls.generator_multiples(lag))


@pytest.fixture(scope="module", params=["plain", "table"])
def setup(request, ctx, points):
    h = ctx.bls12_381_g1_bases_upload(points, 4096)
    if request.param == "table":
        ctx.bases_precompute(h, 0)
    yield h
    ctx.bases_free(h)


def _blobs():
    rng = np.random.default_rng(4844)

    def rand():
        return [int.from_bytes(rng.bytes(32), "big") % bls.R for _ in range(4096)]
    single0, single4095 = [0] * 4096, [0] * 4096
    single0[0], single4095[4095] = SPECIAL, SPECIAL
    mixed = [(bls.R - 1, 0, 1)[i % 3] for i in range(4096)]
    return [rand(), [0] * 4096, [bls.R - 1] * 4096, single0, single4095, mixed, rand(), [1] * 4096]


def _at_tau(vals, lag):
    return sum(v * l for v, l in zip(vals, lag)) % bls.R


def _g(k):
    return bls.compress(bls.generator_multiples([k])[0])


def _proof_at(p_tau, y, z):
    return _g((p_tau - y) * pow((TAU - z) % bls.R, -1, bls.R) % bls.R)


def test_batch_commitments_and_proofs(ctx, setup, lag):
    vals = _blobs()
    blobs = [ref.to_blob(v) for v in vals]
    commitments, proofs = ctx.kzg_blob_to_commitment_and_proof(setup, b"".join(blobs))
    assert len(commitments) == len(proofs) == len(blobs)
    assert commitments[1] == proofs[1] == bytes([0xC0]) + bytes(47)  # the zero blob: identity commitment and quotient
    assert commitments[2] == bls.compress((bls.G1[0], bls.P - bls.G1[1]))  # sum_i L_i = 1, times r - 1
    zs = []
    for b, (v, blob) in enumerate(zip(vals, blobs)):
        p_tau = _at_tau(v, lag)
        assert commitments[b] == _g(p_tau), b
        z = ref.challenge(blob, commitments[b])
        q, y = ref.quotient(v, z)
        assert proofs[b] == _proof_at(p_tau, y, z), b
        # the oracle-driven host path: reference quotient, one MSM per proof
        assert proofs[b] == ctx.bls12_381_g1_msm_resident(setup, ref.to_blob(q), 4096), b
        # one blob per call: the same bytes
        c1, p1 = ctx.kzg_blob_to_commitment_and_proof(setup, blob)
        assert (c1[0], p1[0]) == (commitments[b], proofs[b]), b
        zs.append((z, y))
    # compute_proof at the same challenges, as one batch: the same proofs, and y = the reference's p(z)
    got, ys = ctx.kzg_compute_proof(setup, b"".join(blobs), b"".join(z.to_bytes(32, "big") for z, _ in zs))
    assert got == proofs
    assert [int.from_bytes(y, "big") for y in ys] == [y for _, y in zs]
    assert commitments == ctx.kzg_blob_to_commitment(setup, b"".join(blobs))


def test_compute_proof_in_and_out_of_domain(ctx, setup, lag):
    roots = ref.roots_brp()
    assert roots[0] == 1 and roots[1] == bls.R - 1
    vals = _blobs()
    rng = np.random.default_rng(7594)
    pairs = [(0, roots[0]), (0, roots[1]), (0, roots[77]), (0, roots[4095]), (0, 0), (0, int.from_bytes(rng.bytes(32), "big") % bls.R),
             (5, roots[77]), (3, roots[0]), (4, roots[4095]), (2, roots[1])]
    blobs = b"".join(ref.to_blob(vals[b]) for b, _ in pairs)
    proofs, ys = ctx.kzg_compute_proof(setup, blobs, b"".join(z.to_bytes(32, "big") for _, z in pairs))
    for k, (b, z) in enumerate(pairs):
        v = vals[b]
        q, y = ref.quotient(v, z)
        assert int.from_bytes(ys[k], "big") == y == ref.evaluate_direct(v, z), k
        if z in roots:
            assert y == v[roots.index(z)], k
        assert proofs[k] == _proof_at(_at_tau(v, lag), y, z), k
        assert proofs[k] == ctx.bls12_381_g1_msm_resident(setup, ref.to_blob(q), 4096), k


def test_kzg_settings_run_on_the_device(ctx, points):
    """KzgSettings' proof methods keep their signatures, results and exception types"""
    from ethrex_b200.kzg import KzgSettings
    settings = KzgSettings(ctx, points)
    try:
        vals = _blobs()[0]
        blob = ref.to_blob(vals)
        launches = ctx.launch_count
        c, proof = settings.blob_to_kzg_commitment_and_proof(blob)
        assert ctx.launch_count > launches
        z = settings.compute_challenge(blob, c)
        assert z == ref.challenge(blob, c)
        assert settings.compute_blob_kzg_proof(blob, c) == proof
        p, y = settings.compute_kzg_proof(blob, z)
        assert (p, y) == (proof, ref.quotient(vals, z)[1])
        assert settings.blobs_to_kzg_commitments_and_proofs([blob, blob]) == ([c, c], [proof, proof])
        bad = bls.R.to_bytes(32, "big") + blob[32:]
        with pytest.raises(ValueError):
            settings.compute_kzg_proof(bad, 5)
        with pytest.raises(ValueError):
            settings.compute_kzg_proof(blob, bls.R)
        with pytest.raises(ValueError):
            settings.compute_blob_kzg_proof(bad, c)
        with pytest.raises(eb.B200Error):
            settings.blob_to_kzg_commitment_and_proof(bad)
    finally:
        settings.close()


def test_msm_only_context_composes_the_same_proofs(ctx, setup):
    """KzgSettings over an object that serves only the two MSM calls (scalar-field work in Python) gives the same bytes as
    the one-call device path"""
    from ethrex_b200.kzg import KzgSettings

    class MsmOnly:
        def kzg_blob_to_commitment(self, h, blobs): return ctx.kzg_blob_to_commitment(h, blobs)
        def bls12_381_g1_msm_resident(self, h, scalars, n, flags=F.SCALARS_BE): return ctx.bls12_381_g1_msm_resident(h, scalars, n, flags)

    composed, device = KzgSettings.__new__(KzgSettings), KzgSettings.__new__(KzgSettings)
    composed.ctx, composed.handle, device.ctx, device.handle = MsmOnly(), setup, ctx, setup
    vals = _blobs()
    for blob in (ref.to_blob(vals[0]), ref.to_blob(vals[5])):
        assert composed.blob_to_kzg_commitment_and_proof(blob) == device.blob_to_kzg_commitment_and_proof(blob)
        z = ref.roots_brp()[77]
        assert composed.compute_kzg_proof(blob, z) == device.compute_kzg_proof(blob, z)


def _raw_and_proof(ctx, h, blobs, n, cm, pr):
    return F.lib.b200zk_kzg_blob_to_commitment_and_proof(ctx._h, h, blobs, n, cm, pr)


def _raw_compute(ctx, h, blobs, n, z, pr, y):
    return F.lib.b200zk_kzg_compute_proof(ctx._h, h, blobs, n, z, pr, y)


def test_refusals(ctx, setup):
    good = ref.to_blob(_blobs()[0])
    bad = bytearray(good * 3)
    bad[2 * 131072 + 32 * 4095:2 * 131072 + 32 * 4096] = bls.R.to_bytes(32, "big")  # the last element of the last blob
    n = 3
    cm, pr, y = C.create_string_buffer(b"\xaa" * 48 * n), C.create_string_buffer(b"\xaa" * 48 * n), C.create_string_buffer(b"\xaa" * 32 * n)
    zs = b"".join((5).to_bytes(32, "big") for _ in range(n))
    blob_buf = C.create_string_buffer(bytes(bad))
    assert _raw_and_proof(ctx, setup, blob_buf, n, cm, pr) == F.ERR_NOT_IN_FIELD
    assert b"blob 2" in F.lib.b200zk_last_error(ctx._h)
    assert _raw_compute(ctx, setup, blob_buf, n, zs, pr, y) == F.ERR_NOT_IN_FIELD
    assert b"blob 2" in F.lib.b200zk_last_error(ctx._h)
    assert cm.raw[:-1] == pr.raw[:-1] == b"\xaa" * 48 * n and y.raw[:-1] == b"\xaa" * 32 * n  # nothing written
    # z = r in the second of three pairs
    zbad = (5).to_bytes(32, "big") + bls.R.to_bytes(32, "big") + (7).to_bytes(32, "big")
    assert _raw_compute(ctx, setup, good * 3, n, zbad, pr, y) == F.ERR_NOT_IN_FIELD
    assert b"blob 1" in F.lib.b200zk_last_error(ctx._h)
    assert pr.raw[:-1] == b"\xaa" * 48 * n and y.raw[:-1] == b"\xaa" * 32 * n
    # null pointers with n > 0; n = 0 is a no-op
    assert _raw_and_proof(ctx, setup, None, 1, cm, pr) == F.ERR_INVALID_ARG
    assert _raw_and_proof(ctx, setup, good, 1, cm, None) == F.ERR_INVALID_ARG
    assert _raw_compute(ctx, setup, good, 1, None, pr, y) == F.ERR_INVALID_ARG
    assert _raw_compute(ctx, setup, good, 1, zs, pr, None) == F.ERR_INVALID_ARG
    assert _raw_and_proof(ctx, setup, None, 0, None, None) == F.OK
    assert _raw_compute(ctx, setup, None, 0, None, None, None) == F.OK
    assert ctx.kzg_blob_to_commitment_and_proof(setup, b"") == ([], [])
    # a 1-point BLS12-381 setup, a BN254 handle of 4096 points, an unknown handle
    h1 = ctx.bls12_381_g1_bases_upload(bls.G1_COMPRESSED, 1)
    hb = ctx.g1_bases_upload(bytes(64 * 4096), 4096)
    try:
        for h in (h1, hb, 0xDEAD):
            assert _raw_and_proof(ctx, h, good, 1, cm, pr) == F.ERR_INVALID_ARG
            assert _raw_compute(ctx, h, good, 1, zs, pr, y) == F.ERR_INVALID_ARG
        with pytest.raises(eb.B200Error):
            ctx.kzg_compute_proof(h1, good, zs[:32])
    finally:
        ctx.bases_free(h1)
        ctx.bases_free(hb)
    # the context still works after every refusal
    c, p = ctx.kzg_blob_to_commitment_and_proof(setup, good)
    assert ctx.kzg_compute_proof(setup, good, ref.challenge(good, c[0]).to_bytes(32, "big"))[0] == p
