"""EIP-7594 cell proofs on the device (b200zk_kzg_blob_to_commitment_and_cell_proofs, FK20) over a synthetic known-tau
setup (the mainnet setup is not in the tree): the Lagrange points as in tests/test_gpu_kzg_cells.py plus [tau^i]1 for
i < 4096.  Commitments and proofs are byte-equal to tests/kzg_cells_ref.py's, accepted by the device's own cell-proof
verifier, and malformed input gets its status."""
import ctypes

import numpy as np
import pytest

import bls_ref as bls
import kzg_cells_ref as ref
import kzg_ref

pytestmark = pytest.mark.gpu

import ethrex_b200 as eb  # noqa: E402
from ethrex_b200 import _ffi  # noqa: E402
from ethrex_b200.kzg import KzgSettings  # noqa: E402

TAU = 0x2F1B7C93D4A5E6F708192A3B4C5D6E7F8091A2B3C4D5E6F708192A3B4C5D6E7F % bls.R
IDENTITY = bytes([0xC0]) + bytes(47)
ZERO_BLOB = bytes(131072)
TOP_BLOB = kzg_ref.to_blob([bls.R - 1] * 4096)


def _monomial_blob(e):
    """p = X^e in the blob's evaluation form"""
    return kzg_ref.to_blob([pow(w, e, bls.R) for w in kzg_ref.roots_brp()])


def _blobs(k, seed):
    rng = np.random.default_rng(seed)
    return [kzg_ref.to_blob([int.from_bytes(rng.bytes(32), "big") % bls.R for _ in range(4096)]) for _ in range(k)]


@pytest.fixture(scope="module")
def points():
    return b"".join(bls.compress(p) for p in bls.generator_multiples(bls.lagrange_setup_scalars(TAU)))


@pytest.fixture(scope="module")
def monomial():
    return b"".join(bls.compress(p) for p in bls.generator_multiples([pow(TAU, i, bls.R) for i in range(4096)]))


@pytest.fixture(scope="module")
def g2_points():
    return ref.g2_setup(TAU)


@pytest.fixture(scope="module")
def setups(ctx, points, monomial, g2_points):
    lag = ctx.bls12_381_g1_bases_upload(points, 4096)
    ctx.bases_precompute(lag, 0)
    mono = ctx.bls12_381_g1_bases_upload(monomial, 4096)
    g2 = ctx.bls12_381_g2_bases_upload(g2_points, 65)
    yield lag, mono, g2
    for h in (lag, mono, g2):
        ctx.bases_free(h)


@pytest.fixture(scope="module")
def bundle():
    """24 blobs: the special ones first (zero, all r - 1, X^4095, X^64, X^63), then random; with the oracle's bundle"""
    blobs = [ZERO_BLOB, TOP_BLOB, _monomial_blob(4095), _monomial_blob(64), _monomial_blob(63)] + _blobs(19, seed=7594)
    cs, ps = ref.bundle(blobs, TAU)
    return blobs, cs, ps


def _prove(ctx, setups, blobs):
    return ctx.kzg_blob_to_commitment_and_cell_proofs(setups[0], setups[1], b"".join(blobs))


@pytest.mark.parametrize("k", [1, 6, 24])
def test_matches_oracle(ctx, setups, bundle, k):
    blobs, cs, ps = bundle
    got_c, got_p = _prove(ctx, setups, blobs[:k])
    assert got_c == cs[:k]
    assert got_p == ps[:128 * k]


def test_constant_blobs_give_identity_proofs(ctx, setups, bundle):
    blobs, cs, ps = bundle
    got_c, got_p = _prove(ctx, setups, blobs[:2])
    assert got_c[0] == IDENTITY and got_p == [IDENTITY] * 256


def test_commitments_equal_blob_to_commitment(ctx, setups, bundle):
    blobs = bundle[0][:6]
    assert _prove(ctx, setups, blobs)[0] == ctx.kzg_blob_to_commitment(setups[0], b"".join(blobs))


@pytest.mark.parametrize("k", [1, 6, 24])
def test_device_verifier_accepts(ctx, setups, bundle, k):
    blobs = bundle[0][:k]
    cs, ps = _prove(ctx, setups, blobs)
    assert ctx.kzg_verify_cell_proof_batch(setups[0], setups[2], b"".join(blobs), b"".join(cs), b"".join(ps)) is True
    wrong = ps[:]
    wrong[k * 128 - 1], wrong[k * 128 - 2] = wrong[k * 128 - 2], wrong[k * 128 - 1]
    if wrong != ps:
        assert ctx.kzg_verify_cell_proof_batch(setups[0], setups[2], b"".join(blobs), b"".join(cs), b"".join(wrong)) is False


def test_batch_and_single_calls_agree(ctx, setups, bundle):
    blobs = bundle[0][:6]
    batch = _prove(ctx, setups, blobs)
    assert _prove(ctx, setups, blobs) == batch  # served from the cached table
    for i, blob in enumerate(blobs):
        c, p = _prove(ctx, setups, [blob])
        assert c == [batch[0][i]] and p == batch[1][128 * i:128 * (i + 1)]


def test_statuses(ctx, setups, bundle, monomial):
    lag, mono, g2 = setups
    blobs = bundle[0][5:8]
    bad = bytearray(b"".join(blobs))
    bad[131072 * 2 + 32 * 17:131072 * 2 + 32 * 18] = bls.R.to_bytes(32, "big")
    cm, pr = bytearray(b"\xAA" * 48 * 3), bytearray(b"\xAA" * 128 * 48 * 3)
    st = _ffi.lib.b200zk_kzg_blob_to_commitment_and_cell_proofs(ctx._h, lag, mono, bytes(bad), 3,
                                                                (ctypes.c_char * len(cm)).from_buffer(cm),
                                                                (ctypes.c_char * len(pr)).from_buffer(pr))
    assert st == 2
    assert b"blob 2, element 17" in _ffi.lib.b200zk_last_error(ctx._h)
    assert cm == b"\xAA" * 48 * 3 and pr == b"\xAA" * 128 * 48 * 3  # nothing written
    with pytest.raises(eb.B200Error, match="blob 2, element 17") as e:
        ctx.kzg_blob_to_commitment_and_cell_proofs(lag, mono, bytes(bad))
    assert e.value.status == 2
    small = ctx.bls12_381_g1_bases_upload(monomial[:48 * 4095], 4095)
    freed = ctx.bls12_381_g1_bases_upload(monomial, 4096)
    _prove(ctx, (lag, freed), blobs[:1])  # builds the freed handle's table, so freeing releases it
    ctx.bases_free(freed)
    try:
        for a, b in ((lag, g2), (g2, mono), (lag, small), (small, mono), (lag, freed), (lag, 999999)):
            with pytest.raises(eb.B200Error) as e:
                ctx.kzg_blob_to_commitment_and_cell_proofs(a, b, b"".join(blobs))
            assert e.value.status == 4
    finally:
        ctx.bases_free(small)
    assert ctx.kzg_blob_to_commitment_and_cell_proofs(lag, mono, b"") == ([], [])


def test_kzg_settings_agrees_with_context(ctx, setups, points, monomial, bundle):
    blobs = bundle[0][3:6]
    want = _prove(ctx, setups, blobs)
    s = KzgSettings(ctx, points, g1_monomial=monomial)
    try:
        assert s.blobs_to_commitments_and_cell_proofs(blobs) == want
        assert s.blob_to_commitment_and_cell_proofs(blobs[1]) == (want[0][1], want[1][128:256])
        assert s.blobs_to_commitments_and_cell_proofs([]) == ([], [])
        with pytest.raises(ValueError):
            s.blob_to_commitment_and_cell_proofs(bls.R.to_bytes(32, "big") + blobs[0][32:])
    finally:
        s.close()
    plain = KzgSettings(ctx, points, precompute=False)
    try:
        with pytest.raises(ValueError, match="g1_monomial"):
            plain.blob_to_commitment_and_cell_proofs(blobs[0])
    finally:
        plain.close()
