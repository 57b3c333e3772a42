"""The BLS12-381 pairing check on the device (b200zk_bls12_381_pairing_check_batch) and the G2 bases handle
(b200zk_bls12_381_g2_bases_upload): the reference's EIP-2537 vectors, bilinear products, identities, every status, batching,
and agreement with the independent oracle (tests/bls_pairing_ref.py)."""
import json
import os

import numpy as np
import pytest

import bls_pairing_ref as B
import bls_ref as bls

pytestmark = pytest.mark.gpu

import ethrex_b200 as eb  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
KATS = json.load(open(os.path.join(HERE, "golden", "bls12_pairing_kats.json")))["vectors"]


def _pair(p, q) -> bytes:
    return B.g1_eip2537(p) + B.g2_eip2537(q)


def _g1(k):
    return bls.generator_multiples([k])[0]


def _bilinear_check(rng, k, tamper=False):
    """k pairs (a_i G1, b_i G2) whose product is one: the last pair is (-(sum of the others' a_i b_i) G1, G2)"""
    pairs, acc = [], 0
    for _ in range(k - 1):
        a, b = (int.from_bytes(rng.bytes(32), "big") % bls.R for _ in range(2))
        pairs.append((_g1(a), B.g2_mul(b, B.G2)))
        acc += a * b
    if k:
        pairs.append((_g1(-acc % bls.R + (1 if tamper else 0)), B.G2))
    return b"".join(_pair(p, q) for p, q in pairs)


def test_reference_vectors(ctx):
    res, st = ctx.bls12_381_pairing_check_batch([bytes.fromhex(v["calldata"]) for v in KATS])
    assert res == [v["expected"] for v in KATS] == [0, 0, 1]
    assert st == [0, 0, 0]


@pytest.mark.parametrize("k", range(6))
def test_bilinear_products(ctx, k):
    rng = np.random.default_rng(100 + k)
    good = _bilinear_check(rng, k)
    checks = [good]
    if k:
        checks.append(_bilinear_check(np.random.default_rng(100 + k), k, tamper=True))
    res, st = ctx.bls12_381_pairing_check_batch(checks)
    assert st == [0] * len(checks)
    assert res == ([1, 0] if k else [1])


def test_identity_pairs(ctx):
    g, q = B.G1, B.G2
    checks = [_pair(None, q), _pair(g, None), _pair(None, None), _pair(None, q) + _pair(g, q), _pair(g, q) + _pair(g, B.g2_neg(q)) + _pair(None, None), b""]
    res, st = ctx.bls12_381_pairing_check_batch(checks)
    assert st == [0] * 6
    assert res == [1, 1, 1, 0, 1, 1]


def test_statuses_and_neighbours(ctx):
    g, q = B.G1, B.G2
    valid = _pair(g, q) + _pair(g, B.g2_neg(q))
    x_ge_p = bytes(16) + B.P.to_bytes(48, "big") + B.fp64(g[1]) + B.g2_eip2537(q)
    padding = bytearray(_pair(g, q))
    padding[3] = 1
    g2_pad = bytearray(_pair(g, q))
    g2_pad[128 + 64 * 3 + 5] = 1
    off_g1 = B.fp64(g[0]) + B.fp64((g[1] + 1) % B.P) + B.g2_eip2537(q)
    off_g2 = B.g1_eip2537(g) + B.g2_eip2537((q[0], B.f2_add(q[1], (1, 0))))
    p_out = B.g1_random_point(2537)
    q_out = B.g2_random_point(2537)
    assert not B.g1_in_subgroup(p_out) and not B.g2_in_subgroup(q_out)
    g1_sub = _pair(p_out, q)
    g2_sub = _pair(g, q_out)
    g2_y_ge_p = B.g1_eip2537(g) + B.fp64(q[0][0]) + B.fp64(q[0][1]) + B.fp64(q[1][0] + B.P) + B.fp64(q[1][1])
    cases = [(x_ge_p, 2), (bytes(padding), 2), (bytes(g2_pad), 2), (off_g1, 3), (off_g2, 3), (g1_sub, 3), (g2_sub, 3), (g2_y_ge_p, 2),
             (off_g1 + x_ge_p, 2), (g2_sub + bytes(padding), 2), (valid + off_g2, 3)]
    checks = []
    for bad, _ in cases:
        checks += [valid, bad]
    checks.append(valid)
    res, st = ctx.bls12_381_pairing_check_batch(checks)
    for i, (_, want) in enumerate(cases):
        assert (res[2 * i + 1], st[2 * i + 1]) == (0, want), i
    assert all(res[2 * i] == 1 and st[2 * i] == 0 for i in range(len(cases) + 1))


def test_batch_equals_single_calls(ctx):
    rng = np.random.default_rng(381)
    base = [_bilinear_check(np.random.default_rng(s), 2) for s in range(4)] + [_bilinear_check(np.random.default_rng(s), 2, tamper=True) for s in range(4)]
    checks = [base[int(i)] for i in rng.integers(0, len(base), 256)]
    res, st = ctx.bls12_381_pairing_check_batch(checks)
    singles = [ctx.bls12_381_pairing_check_batch([c]) for c in checks]
    assert res == [r[0][0] for r in singles] and st == [r[1][0] for r in singles]
    assert sorted(set(res)) == [0, 1]


def test_random_checks_agree_with_the_oracle(ctx):
    rng = np.random.default_rng(12381)
    checks, pairs_of = [], []
    for k in range(5):
        ab = [(int(rng.integers(1, 1 << 62)), int(rng.integers(1, 1 << 62))) for _ in range(1 + k % 3)]
        if k % 2:  # make it hold: the last pair cancels the product so far
            ab.append((-sum(a * b for a, b in ab) % bls.R, 1))
        pairs = [(_g1(a), B.g2_mul(b, B.G2)) for a, b in ab]
        checks.append(b"".join(_pair(p, q) for p, q in pairs))
        pairs_of.append(pairs)
    res, st = ctx.bls12_381_pairing_check_batch(checks)
    assert st == [0] * len(checks)
    assert res == [int(B.pairing_check(p)) for p in pairs_of]
    assert res == [0, 1, 0, 1, 0]


def test_g2_upload_statuses_and_refusals(ctx):
    tau = 0x1234567
    q = B.g2_mul(tau, B.G2)
    h = ctx.bls12_381_g2_bases_upload(B.G2_COMPRESSED + B.g2_compress(q) + B.g2_compress(None), 3)
    try:
        with pytest.raises(eb.B200Error) as e:
            ctx.bases_precompute(h, 0)
        assert e.value.status == 4
        for call in (lambda: ctx.g1_msm_resident(h, bytes(32), 1), lambda: ctx.g2_msm_resident(h, bytes(32), 1),
                     lambda: ctx.bls12_381_g1_msm_resident(h, bytes(32), 1), lambda: ctx.kzg_blob_to_commitment(h, bytes(131072)),
                     lambda: ctx.kzg_compute_proof(h, bytes(131072), bytes(32)), lambda: ctx.kzg_blob_to_commitment_and_proof(h, bytes(131072))):
            with pytest.raises(eb.B200Error) as e:
                call()
            assert e.value.status == 4
    finally:
        ctx.bases_free(h)
    x_ge_p = bytearray(B.G2_COMPRESSED)
    x_ge_p[48:] = B.P.to_bytes(48, "big")
    no_c = bytearray(B.G2_COMPRESSED)
    no_c[0] &= 0x7F
    bad_inf = bytes([0xE0]) + bytes(95)
    x = 1
    while B.f2_sqrt(B.f2_add(B.f2_mul(B.f2_sqr((x, 0)), (x, 0)), B.B2)) is not None:
        x += 1
    off = bytearray(bytes(48) + x.to_bytes(48, "big"))
    off[0] |= 0x80
    not_sub = B.g2_compress(B.g2_random_point(4844))
    for pts, want in ((bytes(x_ge_p), 2), (bytes(no_c), 3), (bad_inf, 3), (bytes(off), 3), (not_sub, 3), (B.G2_COMPRESSED + bytes(x_ge_p), 2)):
        with pytest.raises(eb.B200Error) as e:
            ctx.bls12_381_g2_bases_upload(pts, len(pts) // 96)
        assert e.value.status == want, pts.hex()[:8]
    with pytest.raises(eb.B200Error) as e:
        ctx.bls12_381_g2_bases_upload(B.G2_COMPRESSED, 1, flags=0)
    assert e.value.status == 4
