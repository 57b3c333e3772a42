"""MODEXP on the device (b200zk_modexp_batch, precompile 0x05) against Python's `pow` (tests/modexp_ref.py): every size
class edge, even moduli 2^s q and powers of two, carries and borrows through whole lanes, the trivial operands in every
combination, base reduction, Fermat identities for the curve primes, RSA-2048 / 4096 signatures, the 1024/1024/1024 worst
case, a mixed batch against single calls, items over the EIP-7823 bound between valid neighbours, and the argument
refusals and workspace sharing."""
import ctypes as C
import itertools
import random

import pytest

import bls_ref
import modexp_ref as ref
import pyref
import secp256k1_ref as k1
import secp256r1_ref as r1

pytestmark = pytest.mark.gpu

import ethrex_b200 as eb  # noqa: E402
from ethrex_b200 import _ffi as F  # noqa: E402


def check(ctx, items):
    outs, st = ctx.modexp_batch(items)
    want = [ref.expected(it) for it in items]
    for i, (it, (o, s), (wo, ws)) in enumerate(zip(items, zip(outs, st), want)):
        assert (s, o) == (ws, wo), f"item {i}: lengths {[len(x) for x in it]}"
    return outs


def test_class_edges(ctx):
    rng = random.Random(1)
    items = []
    for ml in ref.CLASS_EDGES:
        for odd in (True, False):
            items.append(ref.rand_item(rng, ml, odd=odd))
            items.append(ref.rand_item(rng, ml, base_len=rng.randrange(0, 1025), exp_len=rng.randrange(1, 8), odd=odd))
        # leading zero bytes that keep a modulus in a lower class than its length says
        b, e, m = ref.rand_item(rng, ml, exp_len=4)
        items.append((b, e, bytes(1024 - ml) + m))
    check(ctx, items)


def test_even_moduli(ctx):
    rng = random.Random(2)
    items = []
    for s in (1, 31, 32, 33, 255, 4000):
        for qbits in (1, 7, 64, 300, 8191 - s):
            if qbits <= 0 or s + qbits > 8192:
                continue
            q = rng.getrandbits(qbits) | 1 | (1 << (qbits - 1))
            m = q << s
            ml = (m.bit_length() + 7) // 8
            items.append((ref.rand_bytes(rng, rng.randrange(0, 1025), top=False), ref.rand_bytes(rng, 8), ref.be(m, ml)))
    for k in (0, 1, 8, 31, 32, 33, 255, 256, 257, 1000, 4096, 8191):  # powers of two, up to 2^8191
        m = 1 << k
        items.append((ref.rand_bytes(rng, 64), ref.rand_bytes(rng, 4), ref.be(m, (k + 8) // 8)))
        items.append((ref.be(3, 1), ref.rand_bytes(rng, 1), ref.be(m, (k + 8) // 8)))
    check(ctx, items)


def test_lane_carry_items(ctx):
    """items whose products send carries and borrows through whole lanes (the carry events of tests/bigmod_ref.py,
    through the real kernel), in every class: m = 2^(32N) - 1 with base m - 1, whose Montgomery products reach t = R
    and fold a carry through every lane; m = 2^(32N) - 2^32 + 1 with an all-ones base; and even moduli 2^s q with s on
    lane boundaries, so that m >> s moves whole lanes, and q = 2^(32N - s) - 1 filling the class"""
    rng = random.Random(12)
    items = []
    for bits in (256, 1024, 2048, 4096, 8192):
        n = bits // 8
        m = (1 << bits) - 1
        items += [(ref.be(m - 1, n), b"\x02", ref.be(m, n)), (ref.be(m - 1, n), ref.rand_bytes(rng, 32), ref.be(m, n))]
        items.append((b"\xff" * n, ref.rand_bytes(rng, 32), ref.be((1 << bits) - (1 << 32) + 1, n)))
        for s in (256, 512, 1024, 4096):
            if s < bits:
                m = ((1 << (bits - s)) - 1) << s
                for base in (ref.rand_bytes(rng, n), b"\xff" * n):
                    items.append((base, ref.rand_bytes(rng, 16), ref.be(m, n)))
    outs = check(ctx, items)
    assert outs[0] == ref.be(1, 32)  # (m - 1)^2 = 1


def test_trivial_operands_in_every_combination(ctx):
    bases = [b"", b"\x00", bytes(5), b"\x01", b"\x07", bytes(3) + b"\x05"]
    exps = [b"", b"\x00", bytes(40), b"\x01", bytes(2) + b"\x01", b"\x03"]
    mods = [b"", b"\x00", bytes(33), b"\x01", bytes(4) + b"\x01", b"\x02", b"\x0b", bytes(2) + b"\x0b\x00"]
    items = list(itertools.product(bases, exps, mods))
    outs = check(ctx, items)
    assert outs[items.index((b"\x07", b"", b"\x01"))] == b"\x00"
    assert outs[items.index((b"", b"", b"\x0b"))] == b"\x01"


def test_base_reduction(ctx):
    rng = random.Random(3)
    items = [ref.rand_item(rng, 1, base_len=1024, exp_len=32)]  # a 1024-byte base over a 1-byte modulus
    for ml in (1, 32, 33, 128, 256, 512, 1024):
        m = int.from_bytes(ref.rand_bytes(rng, ml), "big") | 3
        items.append((ref.be(m - 1, ml), b"\x02", ref.be(m, ml)))                    # (m - 1)^2 = 1
        items.append((ref.be(m + rng.getrandbits(64), ml + 8), b"\x05", ref.be(m, ml)))  # b >= m
        ones = b"\xff" * ml
        items.append((ones, ones[:64], ones))                                         # all-ones operands
        items.append((ref.rand_bytes(rng, 1024), ref.rand_bytes(rng, 3), ref.be(m, ml)))
    outs = check(ctx, items)
    assert outs[1] == ref.be(1, 1)


def test_fermat_identities_for_the_curve_primes(ctx):
    rng = random.Random(4)
    items = []
    for p in (pyref.P, pyref.R, bls_ref.P, bls_ref.R, k1.P, k1.N, r1.P, r1.N):
        n = (p.bit_length() + 7) // 8
        for b in (2, 3, rng.randrange(2, p)):
            items.append((ref.be(b, n), ref.be(p - 1, n), ref.be(p, n)))
    outs, st = ctx.modexp_batch(items)
    assert st == [0] * len(items)
    assert all(int.from_bytes(o, "big") == 1 for o in outs)


@pytest.mark.parametrize("bits", [2048, 4096])
def test_rsa_signatures(ctx, bits):
    items, want = ref.rsa_items(random.Random(bits), bits, 16)
    outs, st = ctx.modexp_batch(items)
    assert st == [0] * 16 and outs == want
    assert all(o[:2] == b"\x00\x01" for o in outs)  # PKCS #1 v1.5 encoding


def test_worst_case_item(ctx):
    rng = random.Random(5)
    check(ctx, [(ref.rand_bytes(rng, 1024), ref.rand_bytes(rng, 1024), ref.rand_bytes(rng, 1024))])


def test_mixed_batch_equals_single_calls(ctx):
    items = ref.mixed_items(random.Random(6), 4096)
    outs = check(ctx, items)
    single = [ctx.modexp_batch([it])[0][0] for it in items]
    assert single == outs


def test_over_the_bound(ctx):
    rng = random.Random(8)
    good = [ref.rand_item(rng, ml) for ml in (32, 256, 1024)]
    over = [(bytes(1025), b"\x01", b"\x07"), (b"\x02", bytes(1024) + b"\x01", b"\x07"),
            (b"\x02", b"\x03", bytes(1025) + b"\x07"), (b"\x02", b"\x03", b"\x01" * 2000)]
    items = [x for pair in zip(good + good[:1], over) for x in pair] + good
    outs = check(ctx, items)
    assert [len(o) for o in outs[1:8:2]] == [1, 1, 1026, 2000]


def test_edge_calls_and_refusals(ctx):
    lib, h = F.lib, ctx._h
    fn = lib.b200zk_modexp_batch
    assert ctx.modexp_batch([]) == ([], [])
    assert fn(h, None, None, 0, None, None) == 0
    data = C.create_string_buffer(b"\x03\x05\x07", 3)
    lens = (C.c_uint32 * 3)(1, 1, 1)
    out, st = C.create_string_buffer(1), C.create_string_buffer(1)
    for args in ((None, lens, out, st), (data, None, out, st), (data, lens, None, st), (data, lens, out, None)):
        assert fn(h, args[0], args[1], 1, args[2], args[3]) == F.ERR_INVALID_ARG
        assert b"null" in lib.b200zk_last_error(h)
    assert fn(None, data, lens, 1, out, st) == F.ERR_INVALID_ARG
    # more items than the kernels index: refused before the lengths are read
    assert fn(h, data, lens, 2 ** 32, out, st) == F.ERR_INVALID_ARG
    assert b"2^32" in lib.b200zk_last_error(h)
    assert fn(h, data, lens, 1, out, st) == 0 and out.raw == bytes([pow(3, 5, 7)]) and st.raw == b"\x00"


def test_shares_the_workspace_with_p256():
    """one context alternating MODEXP calls of growing size with P256VERIFY batches (both carve ws_pairing)"""
    rng = random.Random(9)
    c = eb.Context(0)
    try:
        p256 = bytes.fromhex(P256_ITEM)
        for step in range(6):
            items = [ref.rand_item(rng, rng.choice((32, 256, 1024)), exp_len=8) for _ in range(4 << step)]
            outs, st = c.modexp_batch(items)
            assert st == [0] * len(items) and outs == [ref.modexp(*x) for x in items]
            assert c.secp256r1_verify_batch(p256 * (64 << step)) == [True] * (64 << step)
    finally:
        c.close()


def _p256_item() -> str:
    rng = random.Random(10)
    d = rng.randrange(1, r1.N)
    h = rng.getrandbits(256)
    r, s = r1.sign(d, h, rng.randrange(1, r1.N))
    return r1.encode(h, r, s, r1.mul(d, r1.G)).hex()


P256_ITEM = _p256_item()
