"""EIP-7594 cells on the device (b200zk_kzg_compute_cells, b200zk_kzg_verify_cell_proof_batch) against the Python oracle
of tests/kzg_cells_ref.py over the synthetic known-tau setup of tests/test_gpu_kzg_verify.py: the cells are byte-equal,
honest bundles verify, every tampered bundle does not, and malformed input gets its status."""
import numpy as np
import pytest

import bls_pairing_ref as B
import bls_ref as bls
import kzg_cells_ref as ref
import kzg_ref

pytestmark = pytest.mark.gpu

import ethrex_b200 as eb  # noqa: E402
from ethrex_b200.kzg import KzgSettings  # noqa: E402

TAU = 0x2F1B7C93D4A5E6F708192A3B4C5D6E7F8091A2B3C4D5E6F708192A3B4C5D6E7F % bls.R
IDENTITY = bytes([0xC0]) + bytes(47)
ZERO_BLOB = bytes(131072)
TOP_BLOB = kzg_ref.to_blob([bls.R - 1] * 4096)


def _blobs(k, seed):
    rng = np.random.default_rng(seed)
    return [kzg_ref.to_blob([int.from_bytes(rng.bytes(32), "big") % bls.R for _ in range(4096)]) for _ in range(k)]


@pytest.fixture(scope="module")
def points():
    return b"".join(bls.compress(p) for p in bls.generator_multiples(bls.lagrange_setup_scalars(TAU)))


@pytest.fixture(scope="module")
def g2_points():
    return ref.g2_setup(TAU)


@pytest.fixture(scope="module")
def setups(ctx, points, g2_points):
    g1 = ctx.bls12_381_g1_bases_upload(points, 4096)
    ctx.bases_precompute(g1, 0)
    g2 = ctx.bls12_381_g2_bases_upload(g2_points, 65)
    yield g1, g2
    ctx.bases_free(g1)
    ctx.bases_free(g2)


@pytest.fixture(scope="module")
def bundle():
    """24 blobs (the zero blob at 3) with their commitments and 128 cell proofs each, from the oracle"""
    blobs = _blobs(24, seed=7594)
    blobs[3] = ZERO_BLOB
    cs, ps = ref.bundle(blobs, TAU)
    return blobs, cs, ps


def _verify(ctx, setups, blobs, cs, ps):
    return ctx.kzg_verify_cell_proof_batch(setups[0], setups[1], b"".join(blobs), b"".join(cs), b"".join(ps))


def test_compute_cells_matches_oracle(ctx):
    blobs = _blobs(22, seed=1) + [ZERO_BLOB, TOP_BLOB]
    want = [ref.compute_cells(b) for b in blobs]
    assert ctx.kzg_compute_cells(b"".join(blobs)) == want
    for i in (0, 22, 23):
        assert ctx.kzg_compute_cells(blobs[i]) == [want[i]]
    assert ctx.kzg_compute_cells(b"") == []


def test_compute_cells_refuses_elements_out_of_range(ctx):
    blobs = _blobs(3, seed=2)
    bad = bytearray(b"".join(blobs))
    bad[131072 * 2 + 32 * 17:131072 * 2 + 32 * 18] = bls.R.to_bytes(32, "big")
    with pytest.raises(eb.B200Error, match="blob 2, element 17") as e:
        ctx.kzg_compute_cells(bytes(bad))
    assert e.value.status == 2


@pytest.mark.parametrize("k", [1, 6, 24])
def test_bundles_verify(ctx, setups, bundle, k):
    blobs, cs, ps = bundle
    assert _verify(ctx, setups, blobs[:k], cs[:k], ps[:128 * k]) is True


def test_zero_blob_verifies(ctx, setups, bundle):
    blobs, cs, ps = bundle
    assert cs[3] == IDENTITY and ps[128 * 3:128 * 4] == [IDENTITY] * 128
    assert _verify(ctx, setups, [ZERO_BLOB], [IDENTITY], [IDENTITY] * 128) is True


def test_tampered_bundles_fail(ctx, setups, bundle):
    blobs, cs, ps = bundle[0][:6], bundle[1][:6], bundle[2][:128 * 6]
    cases = []
    swapped = ps[:]  # two proofs of one blob
    swapped[128 + 5], swapped[128 + 9] = swapped[128 + 9], swapped[128 + 5]
    cases.append((blobs, cs, swapped))
    moved = ps[:]  # a proof moved to the same cell of another blob
    moved[128 * 4 + 77] = ps[128 * 2 + 77]
    cases.append((blobs, cs, moved))
    ident = ps[:]  # a proof replaced by the identity on a random blob
    ident[128 * 5 + 100] = IDENTITY
    cases.append((blobs, cs, ident))
    cswap = cs[:]  # one commitment swapped between blobs
    cswap[0], cswap[1] = cswap[1], cswap[0]
    cases.append((blobs, cswap, ps))
    changed = blobs[:]  # one blob element changed
    v = (int.from_bytes(blobs[2][32 * 9:32 * 10], "big") + 1) % bls.R
    changed[2] = blobs[2][:32 * 9] + v.to_bytes(32, "big") + blobs[2][32 * 10:]
    cases.append((changed, cs, ps))
    assert [_verify(ctx, setups, *c) for c in cases] == [False] * len(cases)
    assert _verify(ctx, setups, blobs, cs, ps) is True


def test_statuses(ctx, setups, bundle, g2_points):
    blobs, cs, ps = bundle[0][:2], bundle[1][:2], bundle[2][:256]
    bad = bytearray(blobs[1])
    bad[32 * 40:32 * 41] = bls.R.to_bytes(32, "big")
    with pytest.raises(eb.B200Error, match="blob 1, element 40") as e:
        _verify(ctx, setups, [blobs[0], bytes(bad)], cs, ps)
    assert e.value.status == 2
    x_ge_p = bytearray(bls.P.to_bytes(48, "big"))
    x_ge_p[0] |= 0x80
    no_c = bytearray(ps[130])
    no_c[0] &= 0x7F
    not_sub = bls.compress(B.g1_random_point(7))
    for k, point, want in ((131, bytes(x_ge_p), 2), (130, bytes(no_c), 3), (7, not_sub, 3)):
        q = ps[:]
        q[k] = point
        with pytest.raises(eb.B200Error, match=f"proof of blob {k // 128}, cell {k % 128}") as e:
            _verify(ctx, setups, blobs, cs, q)
        assert e.value.status == want
    with pytest.raises(eb.B200Error, match="commitment of blob 1") as e:
        _verify(ctx, setups, blobs, [cs[0], not_sub], ps)
    assert e.value.status == 3
    g1, g2 = setups
    two = ctx.bls12_381_g2_bases_upload(g2_points[:192], 2)
    try:
        for a, b in ((g1, two), (g1, g1), (g2, g2), (g1, 999999)):
            with pytest.raises(eb.B200Error) as e:
                ctx.kzg_verify_cell_proof_batch(a, b, b"".join(blobs), b"".join(cs), b"".join(ps))
            assert e.value.status == 4
    finally:
        ctx.bases_free(two)
    assert ctx.kzg_verify_cell_proof_batch(g1, g2, b"", b"", b"") is True


def test_kzg_settings_agrees_with_context(ctx, setups, points, g2_points, bundle):
    blobs, cs, ps = bundle[0][:3], bundle[1][:3], bundle[2][:384]
    s = KzgSettings(ctx, points, g2_monomial=g2_points)
    try:
        assert s.compute_cells(blobs[0]) == ctx.kzg_compute_cells(blobs[0])[0]
        assert s.verify_cell_kzg_proof_batch(blobs, cs, ps) is True
        assert _verify(ctx, setups, blobs, cs, ps) is True
        wrong = ps[:]
        wrong[200] = ps[201]
        assert s.verify_cell_kzg_proof_batch(blobs, cs, wrong) is False
        assert _verify(ctx, setups, blobs, cs, wrong) is False
        assert s.verify_cell_kzg_proof_batch([], [], []) is True
        with pytest.raises(ValueError):
            s.verify_cell_kzg_proof_batch(blobs, cs, ps[:-1])
        with pytest.raises(ValueError):
            s.verify_cell_kzg_proof_batch(blobs, cs[:2] + [bls.compress(B.g1_random_point(7))], ps)
        with pytest.raises(ValueError):
            s.compute_cells(bls.R.to_bytes(32, "big") + blobs[0][32:])
    finally:
        s.close()
