"""The precompiles' scalar-multiplication chains on the device at the additions that double, cancel or meet the identity
(tests/chain_edges_ref.py builds the inputs and shows on the CPU that each reaches its event): ecMul and the EIP-2537 MSM
terms over raw scalars, the ECDSA ladder of ECRECOVER and P256VERIFY, map-to-curve inputs whose output is the identity, and
the point-evaluation combine.  Every output is compared byte for byte and status for status with the oracles."""
import random

import pytest

import bls12_map_ref as M
import bls12_ops_ref as ops
import bls_ref as bls
import chain_edges_ref as E
import pyref
import secp256k1_ref as k1
import secp256r1_ref as r1

pytestmark = pytest.mark.gpu


# ---- raw-scalar chains ----------------------------------------------------------------------------------------------------
def _points(r, gen, mul, neg, seed):
    p = mul(random.Random(seed).randrange(2, r), gen)
    return [gen, p, neg(p)]


def _scalars(curve):
    return [(k, label) for k, _, _, label in E.scalar_cases(curve)]


def test_ecmul_edges(ctx):
    pts = _points(pyref.R, pyref.G1_GEN, pyref.g1_mul, lambda p: (p[0], -p[1] % pyref.P), 0xB1)
    items = [(p, k, label) for p in pts for k, label in _scalars("bn254_g1")]
    rng = random.Random(0xB2)

    def want(p, k):
        q = pyref.g1_mul(k, p)
        return pyref.g1_to_be(q), 1 if q is None else 0
    for p, k, label in items:  # one call each
        out, st = ctx.bn254_g1_mul_batch(pyref.g1_to_be(p), k.to_bytes(32, "big"))
        assert (out, st[0]) == want(p, k), label
    batch = []  # each between two generic neighbours
    for p, k, _ in items:
        for q, kk in ((p, rng.randrange(1 << 256)), (p, k), (pyref.g1_mul(rng.randrange(1, pyref.R), pts[0]), rng.randrange(1 << 256))):
            batch.append((q, kk))
    out, st = ctx.bn254_g1_mul_batch(b"".join(pyref.g1_to_be(q) for q, _ in batch), b"".join(k.to_bytes(32, "big") for _, k in batch))
    for i, (q, k) in enumerate(batch):
        assert (out[64 * i:64 * i + 64], st[i]) == want(q, k), i
    assert 1 in st and 0 in st


@pytest.mark.parametrize("g", [ops.G1, ops.G2], ids=lambda g: g.name)
def test_msm_term_edges(ctx, g):
    msm = ctx.bls12_381_g1_msm_batch if g is ops.G1 else ctx.bls12_381_g2_msm_batch
    scalars = _scalars("bls12_381_g1")  # the raw-scalar edges of r, then phi's eigenvalues -1, +0, +1
    if g is ops.G2:  # the same edges, then psi's eigenvalue -1, +0, +1
        lam = E.endomorphism_eigenvalues()["bls12_381_g2"][0]
        scalars = [(k, label) for k, label in _scalars("bls12_381_g1") if not label.startswith("lambda")] + [(lam + d, f"psi{d:+d}") for d in (-1, 0, 1)]
    pts = _points(bls.R, g.gen, g.mul, g.neg, 0xB3)
    items = [(p, k, label) for p in pts for k, label in scalars]

    def want(pairs):
        q = g.msm(pairs)
        return g.encode(q), 1 if q is None else 0
    for p, k, label in items:  # one call each
        outs, st = msm([g.calldata([(p, k)])])
        assert (outs[0], st[0]) == want([(p, k)]), label
    rng = random.Random(0xB4)
    calls = []
    for p, k, _ in items:  # between generic neighbours inside one MSM call, all calls in one batch
        calls.append([(g.mul(rng.randrange(1, bls.R), g.gen), rng.randrange(1 << 256)), (p, k), (p, rng.randrange(1 << 256))])
    calls.append([(p, k) for p, k, _ in items])
    outs, st = msm([g.calldata(c) for c in calls])
    for i, c in enumerate(calls):
        assert (outs[i], st[i]) == want(c), i


# ---- the ECDSA ladder ---------------------------------------------------------------------------------------------------------
def test_ecrecover_ladder_edges(ctx):
    rng = random.Random(0xB5)
    sigs, msgs = [], []
    for c in E.ecrecover_cases():
        msg = rng.randbytes(32)
        sigs += [k1.sign(rng.randrange(1, k1.N), msg, rng.randrange(1, k1.N)), c.data[:65]]
        msgs += [msg, c.data[65:]]
    for low_s in (False, True):
        out, st = ctx.secp256k1_ecrecover_batch(b"".join(sigs), b"".join(msgs), low_s=low_s)
        for i, (sig, msg) in enumerate(zip(sigs, msgs)):
            assert (st[i], out[32 * i:32 * i + 32]) == k1.recover(sig, msg, low_s), (i, low_s)
        assert set(st[1::2]) == ({0, 2, 3} if low_s else {0, 3})
    for sig, msg in zip(sigs[1::2], msgs[1::2]):  # one call each
        out, st = ctx.secp256k1_ecrecover_batch(sig, msg)
        assert (st[0], out) == k1.recover(sig, msg)


def test_p256_ladder_edges(ctx):
    rng = random.Random(0xB6)
    items = []
    for c in E.p256_cases():
        q = r1.mul(rng.randrange(1, r1.N), r1.G)
        h, r, s = r1.forge(q, rng.randrange(1, r1.N), rng.randrange(1, r1.N))
        items += [r1.encode(h, r, s, q), c.data]
    want = [r1.verify(x) for x in items]
    assert all(want[0::2]) and True in want[1::2] and False in want[1::2]
    assert ctx.secp256r1_verify_batch(b"".join(items)) == want
    assert [ctx.secp256r1_verify_batch(x)[0] for x in items[1::2]] == want[1::2]


# ---- map-to-curve -------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def maps():
    return E.map_cases()


@pytest.mark.parametrize("group", ["g1", "g2"])
def test_map_to_infinity(ctx, maps, group):
    rng = random.Random(0xB7)
    if group == "g1":
        cases, fn, oracle, size = maps[0], ctx.bls12_381_map_fp_to_g1_batch, M.map_fp_to_g1_bytes, 128
        rand = [M.fp64(rng.randrange(M.P)) for _ in range(16)]
    else:
        cases, fn, oracle, size = maps[1], ctx.bls12_381_map_fp2_to_g2_batch, M.map_fp2_to_g2_bytes, 256
        rand = [M.fp2_64((rng.randrange(M.P), rng.randrange(M.P))) for _ in range(8)]
    items = [c.data for c in cases]
    for j, x in enumerate(rand):  # random u spread through the batch
        items.insert(j * len(items) // len(rand), x)
    out, st = fn(b"".join(items))
    assert set(st) == {0, 1}
    for i, x in enumerate(items):
        assert (out[size * i:size * (i + 1)], st[i]) == (oracle(x) if x in rand else (bytes(size), 1)), i
    for x in rand:
        assert oracle(x)[1] == 0


# ---- point evaluation ---------------------------------------------------------------------------------------------------------
def test_kzg_combine_edges(ctx):
    g2 = ctx.bls12_381_g2_bases_upload(E.G2_SETUP, 2)
    try:
        cases = E.kzg_cases()
        items = [c.data for c in cases]
        res, st = ctx.kzg_verify_proof_batch(g2, *(b"".join(x[a:b] for x in items) for a, b in ((0, 48), (48, 80), (80, 112), (112, 160))))
        assert st == [0] * len(cases)
        assert res == [int(c.params["valid"]) for c in cases]
        for c in cases:  # one call each
            assert ctx.kzg_verify_proof_batch(g2, c.data[:48], c.data[48:80], c.data[80:112], c.data[112:]) == ([int(c.params["valid"])], [0]), c.label
    finally:
        ctx.bases_free(g2)
