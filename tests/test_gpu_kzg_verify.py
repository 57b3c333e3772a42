"""EIP-4844 KZG verification on the device (b200zk_kzg_verify_proof_batch, b200zk_kzg_verify_blob_proof_batch) over the
synthetic known-tau setup of tests/test_gpu_kzg_proof.py: every proof the device's own prover makes verifies, every
tampered one does not, and malformed input gets its status."""
import numpy as np
import pytest

import bls_pairing_ref as B
import bls_ref as bls
import kzg_ref as ref

pytestmark = pytest.mark.gpu

import ethrex_b200 as eb  # noqa: E402
from ethrex_b200.kzg import KzgSettings  # noqa: E402

TAU = 0x2F1B7C93D4A5E6F708192A3B4C5D6E7F8091A2B3C4D5E6F708192A3B4C5D6E7F % bls.R
G2_SETUP = B.G2_COMPRESSED + B.g2_compress(B.g2_mul(TAU, B.G2))
IDENTITY = bytes([0xC0]) + bytes(47)


@pytest.fixture(scope="module")
def points():
    return b"".join(bls.compress(p) for p in bls.generator_multiples(bls.lagrange_setup_scalars(TAU)))


@pytest.fixture(scope="module")
def setups(ctx, points):
    g1 = ctx.bls12_381_g1_bases_upload(points, 4096)
    ctx.bases_precompute(g1, 0)
    g2 = ctx.bls12_381_g2_bases_upload(G2_SETUP, 2)
    yield g1, g2
    ctx.bases_free(g1)
    ctx.bases_free(g2)


def _blobs(k, seed=4844):
    rng = np.random.default_rng(seed)
    out = [ref.to_blob([int.from_bytes(rng.bytes(32), "big") % bls.R for _ in range(4096)]) for _ in range(k)]
    return out


@pytest.fixture(scope="module")
def items(ctx, setups):
    """(commitment, z, y, proof) from the device prover: random blobs at their challenges, the zero blob, z in the domain"""
    g1, _ = setups
    blobs = _blobs(3) + [bytes(131072)]
    cs, ps = ctx.kzg_blob_to_commitment_and_proof(g1, b"".join(blobs))
    assert cs[3] == ps[3] == IDENTITY
    out = []
    for blob, c, p in zip(blobs, cs, ps):
        z = ref.challenge(blob, c)
        out.append((c, z.to_bytes(32, "big"), ref.quotient(ref.blob_values(blob), z)[1].to_bytes(32, "big"), p))
    roots = ref.roots_brp()
    zs = [roots[0], roots[77], 12345]
    proofs, ys = ctx.kzg_compute_proof(g1, b"".join(blobs[:1] * 3), b"".join(z.to_bytes(32, "big") for z in zs))
    for z, p, y in zip(zs, proofs, ys):
        out.append((cs[0], z.to_bytes(32, "big"), y, p))
    return out


def _verify(ctx, g2, items):
    return ctx.kzg_verify_proof_batch(g2, *(b"".join(it[k] for it in items) for k in range(4)))


def test_device_proofs_verify(ctx, setups, items):
    res, st = _verify(ctx, setups[1], items)
    assert st == [0] * len(items) and res == [1] * len(items)


@pytest.mark.parametrize("field", range(4))
def test_tampered_items_fail_alone(ctx, setups, items, field):
    bad = []
    for k, it in enumerate(items):
        it = list(it)
        if k % 2:
            if field in (1, 2):  # z or y + 1
                it[field] = ((int.from_bytes(it[field], "big") + 1) % bls.R).to_bytes(32, "big")
            else:  # another valid point: the generator
                it[field] = bls.G1_COMPRESSED
        bad.append(tuple(it))
    res, st = _verify(ctx, setups[1], bad)
    assert st == [0] * len(items)
    # the zero blob's proof (identity commitment and proof, y = 0) opens at every z: only its z may change unnoticed
    assert res == [1 if k % 2 == 0 or (field == 1 and items[k][0] == IDENTITY) else 0 for k in range(len(items))]
    assert res.count(0) >= 2


def test_wrong_tau_rejects(ctx, items):
    g2 = ctx.bls12_381_g2_bases_upload(B.G2_COMPRESSED + B.g2_compress(B.g2_mul(TAU + 1, B.G2)), 2)
    try:
        res, st = _verify(ctx, g2, items)
        # the zero blob's identity commitment and proof open under every setup
        assert st == [0] * len(items) and res == [int(it[0] == IDENTITY) for it in items] and sum(res) == 1
    finally:
        ctx.bases_free(g2)


def test_statuses(ctx, setups, items):
    c, z, y, p = items[0]
    x_ge_p = bytearray(bls.P.to_bytes(48, "big"))
    x_ge_p[0] |= 0x80
    no_c = bytearray(c)
    no_c[0] &= 0x7F
    x = 1
    while pow((x ** 3 + 4) % bls.P, (bls.P - 1) // 2, bls.P) == 1:
        x += 1
    off = bytearray(x.to_bytes(48, "big"))
    off[0] |= 0x80
    not_sub = bls.compress(B.g1_random_point(7))
    r = bls.R.to_bytes(32, "big")
    cases = [((c, r, y, p), 2), ((c, z, r, p), 2), ((bytes(x_ge_p), z, y, p), 2), ((c, z, y, bytes(x_ge_p)), 2), ((bytes(no_c), z, y, p), 3),
             ((c, z, y, bytes(off)), 3), ((not_sub, z, y, p), 3), ((c, z, y, not_sub), 3), ((bytes(off), r, y, p), 2)]
    batch = []
    for it, _ in cases:
        batch += [items[0], it]
    res, st = _verify(ctx, setups[1], batch + [items[1]])
    assert st == sum(([0, want] for _, want in cases), []) + [0]
    assert res == [1, 0] * len(cases) + [1]


def test_setup_refusals(ctx, setups, items):
    g1, g2 = setups
    not_gen = ctx.bls12_381_g2_bases_upload(B.g2_compress(B.g2_mul(2, B.G2)) + B.G2_COMPRESSED, 2)
    one = ctx.bls12_381_g2_bases_upload(B.G2_COMPRESSED, 1)
    try:
        for h in (g1, not_gen, one, 999999):
            with pytest.raises(eb.B200Error) as e:
                _verify(ctx, h, items[:1])
            assert e.value.status == 4
            with pytest.raises(eb.B200Error) as e:
                ctx.kzg_verify_blob_proof_batch(h, b"", b"", b"")
            assert e.value.status == 4
    finally:
        ctx.bases_free(not_gen)
        ctx.bases_free(one)


@pytest.mark.parametrize("k", [1, 6, 9])
def test_blob_batches(ctx, setups, k):
    g1, g2 = setups
    blobs = _blobs(k, seed=k)
    if k == 9:
        blobs[4] = bytes(131072)
    cs, ps = ctx.kzg_blob_to_commitment_and_proof(g1, b"".join(blobs))
    joined = b"".join(blobs), b"".join(cs), b"".join(ps)
    assert ctx.kzg_verify_blob_proof_batch(g2, *joined) is True
    tampered = ps[:]
    tampered[k // 2] = bls.G1_COMPRESSED
    assert ctx.kzg_verify_blob_proof_batch(g2, joined[0], joined[1], b"".join(tampered)) is False
    if k > 1:
        swapped = ps[:]
        swapped[0], swapped[1] = swapped[1], swapped[0]
        assert ctx.kzg_verify_blob_proof_batch(g2, joined[0], joined[1], b"".join(swapped)) is False
        bad = bytearray(joined[0])
        bad[131072 * (k - 1) + 32 * 5:131072 * (k - 1) + 32 * 6] = bls.R.to_bytes(32, "big")
        with pytest.raises(eb.B200Error, match=f"blob {k - 1}, element 5") as e:
            ctx.kzg_verify_blob_proof_batch(g2, bytes(bad), joined[1], joined[2])
        assert e.value.status == 2
        with pytest.raises(eb.B200Error, match="proof of blob 1") as e:
            ctx.kzg_verify_blob_proof_batch(g2, joined[0], joined[1], joined[2][:48] + bls.compress(B.g1_random_point(9)) + joined[2][96:])
        assert e.value.status == 3
    assert ctx.kzg_verify_blob_proof_batch(g2, b"", b"", b"") is True


def test_kzg_settings_verify(ctx, points, items):
    s = KzgSettings(ctx, points, g2_monomial=G2_SETUP)
    try:
        c, z, y, p = items[0]
        assert s.verify_kzg_proof(c, z, y, p) is True
        assert s.verify_kzg_proof(c, int.from_bytes(z, "big"), int.from_bytes(y, "big"), p) is True
        assert s.verify_kzg_proof(c, z, y, bls.G1_COMPRESSED) is False
        with pytest.raises(ValueError):
            s.verify_kzg_proof(c, bls.R, y, p)
        with pytest.raises(ValueError):
            s.verify_kzg_proof(bls.compress(B.g1_random_point(7)), z, y, p)
        blobs = _blobs(2, seed=77)
        pairs = [s.blob_to_kzg_commitment_and_proof(b) for b in blobs]
        assert s.verify_blob_kzg_proof(blobs[0], *pairs[0]) is True
        assert s.verify_blob_kzg_proof(blobs[0], pairs[0][0], pairs[1][1]) is False
        assert s.verify_blob_kzg_proof_batch(blobs, [q[0] for q in pairs], [q[1] for q in pairs]) is True
        assert s.verify_blob_kzg_proof_batch([], [], []) is True
        with pytest.raises(ValueError):
            s.verify_blob_kzg_proof(bls.R.to_bytes(32, "big") + blobs[0][32:], *pairs[0])
    finally:
        s.close()
    plain = KzgSettings(ctx, points, precompute=False)
    try:
        with pytest.raises(ValueError):
            plain.verify_kzg_proof(c, z, y, p)
    finally:
        plain.close()
