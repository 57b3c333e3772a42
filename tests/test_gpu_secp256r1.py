"""P-256 signature verification on the device (b200zk_secp256r1_verify_batch, P256VERIFY of EIP-7951): OpenSSL
signatures (through the `cryptography` package) and their high-s twins, tampered items, the constructed edges of the
oracle (tests/secp256r1_ref.py) between valid neighbours, public-key, signature and hash edges, batches against single
calls, the argument refusals, a 2^16 batch, repeated calls on a fresh context (the cached table of G multiples), and one
context alternating secp256k1 recovery and P-256 verification."""
import ctypes as C
import random

import pytest
from cryptography.hazmat.primitives import hashes
from cryptography.hazmat.primitives.asymmetric import ec, utils

import secp256k1_ref as k1
import secp256r1_ref as ref

pytestmark = pytest.mark.gpu

import ethrex_b200 as eb  # noqa: E402
from ethrex_b200 import _ffi as F  # noqa: E402

P, N = ref.P, ref.N


def crypto_item(rng) -> bytes:
    key = ec.derive_private_key(rng.randrange(1, N), ec.SECP256R1())
    digest = rng.randbytes(32)
    r, s = utils.decode_dss_signature(key.sign(digest, ec.ECDSA(utils.Prehashed(hashes.SHA256()))))
    pub = key.public_key().public_numbers()
    return ref.encode(int.from_bytes(digest, "big"), r, s, (pub.x, pub.y))


def flip(inp: bytes, field: int, bit: int) -> bytes:
    b = bytearray(inp)
    b[32 * field + 31 - bit // 8] ^= 1 << (bit % 8)
    return bytes(b)


def with_word(inp: bytes, field: int, value: int) -> bytes:
    return inp[:32 * field] + value.to_bytes(32, "big") + inp[32 * field + 32:]


@pytest.fixture(scope="module")
def signed():
    rng = random.Random(1)
    return [crypto_item(rng) for _ in range(4096)]


def test_openssl_signatures_and_high_s_twins(ctx, signed):
    assert ctx.secp256r1_verify_batch(b"".join(signed)) == [True] * len(signed)
    assert ctx.secp256r1_verify_batch(b"".join(ref.high_s(x) for x in signed)) == [True] * len(signed)


def test_bit_flip_in_each_field(ctx, signed):
    """every item tampered in each of its five words; the oracle (about 10 ms an item in Python) confirms 256 per word"""
    rng = random.Random(2)
    for field in range(5):
        items = [flip(x, field, rng.randrange(256)) for x in signed]
        assert not any(ref.verify(items[i]) for i in rng.sample(range(len(items)), 256))
        assert ctx.secp256r1_verify_batch(b"".join(items)) == [False] * len(items)


def test_constructed_cases_between_valid_neighbours(ctx, signed):
    items, want = [], []
    for i, (_, inp, exp) in enumerate(ref.constructed_cases()):
        items += [signed[i], inp]
        want += [True, exp]
    assert want == [True if i % 2 == 0 else ref.verify(x) for i, x in enumerate(items)]
    got = ctx.secp256r1_verify_batch(b"".join(items))
    assert got == want
    cases = {name: g for (name, _, _), g in zip(ref.constructed_cases(), got[1::2])}
    assert cases["x_above_n"] and cases["equal_points_2g"]


def test_public_key_edges(ctx, signed):
    base = signed[0]
    h, r, s, qx, qy = ref.decode(base)
    # a small-x key whose canonical form verifies, then the same key with qx + p (non-canonical)
    small = next(ref.lift_x(x) for x in range(1, 1000) if ref.lift_x(x) is not None)
    sh, sr, ss = ref.forge(small, 0x1357, 0x2468)
    good_small = ref.encode(sh, sr, ss, small)
    items = [with_word(base, 3, P), with_word(base, 4, P), with_word(base, 3, 2**256 - 1), with_word(base, 4, 2**256 - 1),
             ref.encode(sh, sr, ss, (small[0] + P, small[1])), ref.encode(h, r, s, (0, 0)), with_word(base, 4, (qy + 1) % P), ref.encode(h, r, s, ref.neg((qx, qy)))]
    assert ctx.secp256r1_verify_batch(good_small + base) == [True, True]
    assert ctx.secp256r1_verify_batch(b"".join(items)) == [False] * len(items)
    assert [ref.verify(x) for x in items] == [False] * len(items)


def test_signature_edges(ctx, signed):
    base = signed[1]
    items = [with_word(base, f, v) for f in (1, 2) for v in (0, N, 2**256 - 1)]
    assert ctx.secp256r1_verify_batch(b"".join(items)) == [False] * len(items)


def test_hash_edges(ctx):
    rng = random.Random(3)
    q = ref.mul(0xABCDEF, ref.G)
    items, want = [], []
    for h in (N, N + 1, 2**256 - 1, rng.randrange(N, 2**256)):  # h >= n verifies exactly when h - n does
        r, s = ref.sign(0xABCDEF, h - N, rng.randrange(1, N))
        for hh in (h, h - N):
            items.append(ref.encode(hh, r, s, q))
            want.append(True)
        items.append(ref.encode(h ^ 1, r, s, q))
        want.append(ref.verify(items[-1]))
    r, s = ref.sign(0xABCDEF, 0, rng.randrange(1, N))  # h = 0: u1 = 0, the G term is empty
    items += [ref.encode(0, r, s, q), ref.encode(N, r, s, q), ref.encode(1, r, s, q)]
    want += [ref.verify(x) for x in items[-3:]]
    assert want[-3:] == [True, True, False]
    assert ctx.secp256r1_verify_batch(b"".join(items)) == want


def test_batch_equals_single_calls(ctx, signed):
    rng = random.Random(4)
    items = signed[:16] + [flip(x, rng.randrange(5), rng.randrange(256)) for x in signed[16:24]]
    items += [inp for _, inp, _ in ref.constructed_cases()]
    batch = ctx.secp256r1_verify_batch(b"".join(items))
    assert [ctx.secp256r1_verify_batch(x)[0] for x in items] == batch


def test_refusals(ctx, signed):
    lib, h = F.lib, ctx._h
    inp = C.create_string_buffer(signed[0], 160)
    res = C.create_string_buffer(1)
    fn = lib.b200zk_secp256r1_verify_batch
    assert fn(h, None, 0, None) == 0
    assert fn(h, None, 1, res) == F.ERR_INVALID_ARG
    assert b"null" in lib.b200zk_last_error(h)
    assert fn(h, inp, 1, None) == F.ERR_INVALID_ARG
    assert fn(None, inp, 1, res) == F.ERR_INVALID_ARG
    assert fn(h, inp, 1, res) == 0 and res.raw[0] == 1
    assert ctx.secp256r1_verify_batch(b"") == []
    for n in (1, 159, 161, 319):
        with pytest.raises(eb.B200Error):
            ctx.secp256r1_verify_batch(bytes(n))


def test_large_batch_spot_checked(ctx, signed):
    rng = random.Random(5)
    n = 1 << 16
    items = [signed[i % len(signed)] if i % 3 else flip(signed[i % len(signed)], i % 5, rng.randrange(256)) for i in range(n)]
    got = ctx.secp256r1_verify_batch(b"".join(items))
    assert len(got) == n
    for i in rng.sample(range(n), 256):
        assert got[i] == ref.verify(items[i]), i
    assert got == [i % 3 != 0 for i in range(n)]


def test_fresh_context_repeats_results(signed):
    """a context of its own, so its first call is the one that builds the table"""
    items = b"".join(signed[:32] + [flip(x, 0, 7) for x in signed[32:64]])
    c = eb.Context(0)
    try:
        first = c.secp256r1_verify_batch(items)  # builds the table of G multiples
        second = c.secp256r1_verify_batch(items)
    finally:
        c.close()
    assert first == second == [True] * 32 + [False] * 32


def test_alternating_with_secp256k1_recovery(signed):
    rng = random.Random(6)
    sigs, msgs, want = [], [], []
    for _ in range(32):
        digest = rng.randbytes(32)
        priv = rng.randrange(1, k1.N)
        sig = k1.sign(priv, digest, rng.randrange(1, k1.N))
        sigs.append(sig); msgs.append(digest); want.append(k1.recover(sig, digest)[1])
    p256 = b"".join(signed[:64])
    c = eb.Context(0)
    try:
        for first in ("k1", "r1", "k1", "r1"):
            if first == "k1":
                out, st = c.secp256k1_ecrecover_batch(b"".join(sigs), b"".join(msgs))
                assert st == [0] * 32 and out == b"".join(want)
            else:
                assert c.secp256r1_verify_batch(p256) == [True] * 64
    finally:
        c.close()
