"""secp256k1 signer recovery on the device (b200zk_secp256k1_ecrecover_batch): `cryptography` signatures byte-equal to
the oracle (tests/secp256k1_ref.py) and to the signer's own key, the ethrex L1 genesis keys, every status between valid
neighbours, the low-s flag, batches against single calls, the argument refusals, a 2^16 batch and repeated calls on one
context (the cached table of G multiples)."""
import ctypes as C
import hashlib
import json
import os
import random

import pytest
from cryptography.hazmat.primitives import hashes
from cryptography.hazmat.primitives.asymmetric import ec, utils

import secp256k1_ref as ref

pytestmark = pytest.mark.gpu

import ethrex_b200 as eb  # noqa: E402
from ethrex_b200 import _ffi as F  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
N = ref.N


def crypto_item(rng):
    """(sig, digest, signer's keccak256(X | Y)) from a `cryptography` signature; recid found with the oracle"""
    key = ec.derive_private_key(rng.randrange(1, N), ec.SECP256K1())
    digest = rng.randbytes(32)
    r, s = utils.decode_dss_signature(key.sign(digest, ec.ECDSA(utils.Prehashed(hashes.SHA256()))))
    pub = key.public_key().public_numbers()
    want = ref.address_hash((pub.x, pub.y))
    for recid in (0, 1):
        sig = r.to_bytes(32, "big") + s.to_bytes(32, "big") + bytes([recid])
        if ref.recover(sig, digest) == (ref.OK, want):
            return sig, digest, want
    raise AssertionError("no recid recovers the signer")


def run(ctx, items, low_s=False):
    """items: [(sig, msg)] -> ([32 bytes per item], [status])"""
    out, st = ctx.secp256k1_ecrecover_batch(b"".join(s for s, _ in items), b"".join(m for _, m in items), low_s)
    return [out[32 * i:32 * i + 32] for i in range(len(items))], st


def test_cryptography_signatures(ctx):
    rng = random.Random(1)
    items = [crypto_item(rng) for _ in range(4096)]
    out, st = run(ctx, [(s, m) for s, m, _ in items])
    assert st == [0] * len(items)
    assert out == [w for _, _, w in items]
    assert {s[64] for s, _, _ in items} == {0, 1}


def test_genesis_keys(ctx):
    keys = json.load(open(os.path.join(HERE, "golden", "secp256k1_l1_keys.json")))["keys"]
    rng = random.Random(2)
    items, want = [], []
    for k in keys:
        digest = hashlib.sha256(k["address"].encode()).digest()
        sig = ref.low_s(ref.sign(int(k["private_key"], 16), digest, rng.randrange(1, N)))
        items.append((sig, digest))
        want.append(k["address"])
    out, st = run(ctx, items, low_s=True)
    assert st == [0] * len(keys)
    assert [o[12:].hex() for o in out] == want


def test_every_status_between_valid_neighbours(ctx):
    rng = random.Random(3)
    cases = ref.status_cases()
    for low_s in (False, True):
        items, want = [], []
        for _, sig, msg, flag, expected in cases:
            if flag != low_s:
                continue
            good = ref.sign(rng.randrange(1, N), rng.randbytes(32), rng.randrange(1, N))
            good = ref.low_s(good) if low_s else good
            for s, m in ((good, rng.randbytes(32)), (sig, msg)):
                items.append((s, m))
                want.append(ref.recover(s, m, low_s))
            assert want[-1][0] == expected
        items.append(items[0]); want.append(want[0])
        out, st = run(ctx, items, low_s)
        assert list(zip(st, out)) == want
        assert {w[0] for w in want} == {c[4] for c in cases if c[3] == low_s}


def test_low_s_flag_changes_only_high_s_items(ctx):
    rng = random.Random(4)
    items = [(ref.sign(rng.randrange(1, N), m, rng.randrange(1, N)), m) for m in (rng.randbytes(32) for _ in range(256))]
    high = [int.from_bytes(s[32:64], "big") > ref.N_HALF for s, _ in items]
    assert 50 < sum(high) < 206
    out0, st0 = run(ctx, items)
    out1, st1 = run(ctx, items, low_s=True)
    assert st0 == [0] * len(items)
    for h, o0, s1, o1 in zip(high, out0, st1, out1):
        assert (s1, o1) == ((2, bytes(32)) if h else (0, o0))


def test_batch_equals_single_calls(ctx):
    rng = random.Random(5)
    items = [(ref.sign(rng.randrange(1, N), m, rng.randrange(1, N)), m) for m in (rng.randbytes(32) for _ in range(24))]
    items += [(sig, msg) for _, sig, msg, _, _ in ref.status_cases()]
    out, st = run(ctx, items)
    for i, it in enumerate(items):
        o1, s1 = run(ctx, [it])
        assert (o1[0], s1[0]) == (out[i], st[i])


def test_refusals(ctx):
    lib, h = F.lib, ctx._h
    sig = C.create_string_buffer(ref.sign(7, bytes(32), 11), 65)
    msg = C.create_string_buffer(bytes(32), 32)
    out, st = C.create_string_buffer(32), C.create_string_buffer(1)
    fn = lib.b200zk_secp256k1_ecrecover_batch
    assert fn(h, None, None, 0, 0, None, None) == 0
    assert fn(h, None, msg, 1, 0, out, st) == F.ERR_INVALID_ARG
    assert fn(h, sig, None, 1, 0, out, st) == F.ERR_INVALID_ARG
    assert fn(h, sig, msg, 1, 0, None, st) == F.ERR_INVALID_ARG
    assert fn(h, sig, msg, 1, 0, out, None) == F.ERR_INVALID_ARG
    assert b"null" in lib.b200zk_last_error(h)
    assert fn(h, sig, msg, 1, 2, out, st) == F.ERR_INVALID_ARG
    assert b"flag" in lib.b200zk_last_error(h)
    assert fn(h, sig, msg, 0, 0x80000000, out, st) == F.ERR_INVALID_ARG
    assert fn(None, sig, msg, 1, 0, out, st) == F.ERR_INVALID_ARG
    assert fn(h, sig, msg, 1, F.ECRECOVER_LOW_S, out, st) == 0 and st.raw[0] == ref.recover(sig.raw, bytes(32), True)[0]
    assert ctx.secp256k1_ecrecover_batch(b"", b"") == (b"", [])
    for sigs, msgs in ((bytes(64), bytes(32)), (bytes(65), bytes(31)), (bytes(130), bytes(32))):
        with pytest.raises(eb.B200Error):
            ctx.secp256k1_ecrecover_batch(sigs, msgs)


def test_large_batch_spot_checked(ctx):
    rng = random.Random(6)
    n = 1 << 16
    sigs = bytearray()
    for _ in range(n):
        sigs += rng.randrange(1, N).to_bytes(32, "big") + rng.randrange(1, N).to_bytes(32, "big") + bytes([rng.randrange(2)])
    msgs = rng.randbytes(32 * n)
    out, st = ctx.secp256k1_ecrecover_batch(bytes(sigs), msgs)
    assert len(out) == 32 * n and 0.3 < st.count(0) / n < 0.7 and set(st) == {0, 3}  # about half the x have a curve point
    for i in rng.sample(range(n), 256):
        assert (st[i], out[32 * i:32 * i + 32]) == ref.recover(bytes(sigs[65 * i:65 * i + 65]), msgs[32 * i:32 * i + 32])


def test_fresh_context_repeats_bytes(ctx):
    """a context of its own, so its first call is the one that builds the table (ctx only ensures a device)"""
    rng = random.Random(7)
    items = [crypto_item(rng) for _ in range(64)]
    sigs, msgs = b"".join(s for s, _, _ in items), b"".join(m for _, m, _ in items)
    c = eb.Context(0)
    try:
        first = c.secp256k1_ecrecover_batch(sigs, msgs)  # builds the table of G multiples
        second = c.secp256k1_ecrecover_batch(sigs, msgs)
    finally:
        c.close()
    assert first == second
    assert first == (b"".join(w for _, _, w in items), [0] * len(items))
