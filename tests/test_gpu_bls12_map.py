"""EIP-2537 map-to-curve on the device (b200zk_bls12_381_map_fp_to_g1_batch / _map_fp2_to_g2_batch): every output compared
byte-for-byte with the RFC 9380 oracle (tests/bls12_map_ref.py) on random inputs, SSWU's exceptional inputs and the sgn0
branches, the reference's FP2_ZERO_MAPPED_TO_G2, status 2 with neighbours intact, batches against single calls, the
argument refusals, and the outputs accepted by the subgroup-checking EIP-2537 MSM."""
import ctypes as C
import json
import os
import random

import pytest

import bls12_map_ref as M
import bls_pairing_ref as B
from test_bls12_map_host import g1_exceptional, g2_exceptional

pytestmark = pytest.mark.gpu

import ethrex_b200 as eb  # noqa: E402
from ethrex_b200 import _ffi as F  # noqa: E402

P = M.P
HERE = os.path.dirname(os.path.abspath(__file__))


class G1:
    size, out = 64, 128
    enc = staticmethod(M.fp64)
    oracle = staticmethod(M.map_fp_to_g1_bytes)

    @staticmethod
    def call(ctx, data):
        return ctx.bls12_381_map_fp_to_g1_batch(data)

    @staticmethod
    def rand(rng):
        return rng.randrange(P)

    @staticmethod
    def edges():
        return g1_exceptional() + [1, P - 1, 2, (P - 1) // 2, (P + 1) // 2]


class G2:
    size, out = 128, 256
    enc = staticmethod(M.fp2_64)
    oracle = staticmethod(M.map_fp2_to_g2_bytes)

    @staticmethod
    def call(ctx, data):
        return ctx.bls12_381_map_fp2_to_g2_batch(data)

    @staticmethod
    def rand(rng):
        return rng.randrange(P), rng.randrange(P)

    @staticmethod
    def edges():
        # c0 = 0 or c1 = 0 take each side of sgn0's c0 = 0 branch
        return g2_exceptional() + [(1, 0), (0, 1), (P - 1, 0), (0, P - 1), (2, 0), (0, 2), (P - 1, P - 1), (1, 1), (0, 7), (7, 0)]


GROUPS = [G1, G2]


def _run(ctx, g, encs):
    out, st = g.call(ctx, b"".join(encs))
    return [out[g.out * i:g.out * (i + 1)] for i in range(len(encs))], st


@pytest.mark.parametrize("g", GROUPS, ids=lambda g: g.__name__)
def test_random_and_edge_inputs_match_the_oracle(ctx, g):
    rng = random.Random(0x2537 + g.size)
    us = g.edges() + [g.rand(rng) for _ in range(256)]
    encs = [g.enc(u) for u in us]
    outs, st = _run(ctx, g, encs)
    for i, e in enumerate(encs):
        assert (outs[i], st[i]) == g.oracle(e), us[i]
    assert set(st) == {0}


def test_zero_fp2_is_the_reference_vector(ctx):
    kat = json.load(open(os.path.join(HERE, "golden", "bls12_map_kats.json")))["vectors"][0]
    out, st = ctx.bls12_381_map_fp2_to_g2_batch(bytes.fromhex(kat["input"]))
    assert (out, st) == (bytes.fromhex(kat["expected"]), [0])


def _bad_fields():
    good = M.fp64(0x1234)
    return [bytes([1]) + good[1:], good[:15] + bytes([0x80]) + good[16:], M.fp64(P), bytes(16) + b"\xff" * 48]


@pytest.mark.parametrize("g", GROUPS, ids=lambda g: g.__name__)
def test_status_2_with_neighbours_intact(ctx, g):
    rng = random.Random(7 + g.size)
    bads = _bad_fields()
    if g is G2:
        fine = M.fp64(99)
        bads = [b + fine for b in bads] + [fine + b for b in bads]
    encs, want = [], []
    for b in bads:
        good = g.enc(g.rand(rng))
        encs += [good, b]
        want += [g.oracle(good), (bytes(g.out), 2)]
    encs.append(g.enc(g.rand(rng)))
    want.append(g.oracle(encs[-1]))
    outs, st = _run(ctx, g, encs)
    assert list(zip(outs, st)) == want


@pytest.mark.parametrize("g", GROUPS, ids=lambda g: g.__name__)
def test_batch_equals_single_calls(ctx, g):
    rng = random.Random(11 + g.size)
    pool = [g.enc(u) for u in g.edges()[:4]] + [g.enc(g.rand(rng)) for _ in range(4)] + _bad_fields()[:2 if g is G1 else 0]
    if g is G2:
        pool += [b + M.fp64(3) for b in _bad_fields()[:2]]
    encs = [pool[rng.randrange(len(pool))] for _ in range(150)]
    outs, st = _run(ctx, g, encs)
    for i, e in enumerate(encs):
        o1, s1 = _run(ctx, g, [e])
        assert (outs[i], st[i]) == (o1[0], s1[0]), i
    assert set(st) == {0, 2}


@pytest.mark.parametrize("g", GROUPS, ids=lambda g: g.__name__)
def test_outputs_pass_the_subgroup_checking_msm(ctx, g):
    rng = random.Random(13 + g.size)
    encs = [g.enc(u) for u in g.edges()[:3]] + [g.enc(g.rand(rng)) for _ in range(5)]
    outs, st = _run(ctx, g, encs)
    assert st == [0] * len(encs)
    msm = ctx.bls12_381_g1_msm_batch if g is G1 else ctx.bls12_381_g2_msm_batch
    mo, ms = msm([o + (1).to_bytes(32, "big") for o in outs])
    assert ms == [0] * len(encs) and mo == outs


@pytest.mark.parametrize("g", GROUPS, ids=lambda g: g.__name__)
def test_refusals(ctx, g):
    lib, h = F.lib, ctx._h
    fn = lib.b200zk_bls12_381_map_fp_to_g1_batch if g is G1 else lib.b200zk_bls12_381_map_fp2_to_g2_batch
    inp = C.create_string_buffer(g.enc(g.edges()[3]), g.size)
    out, st = C.create_string_buffer(g.out), C.create_string_buffer(1)
    assert fn(h, None, 0, None, None) == 0
    assert fn(h, None, 1, out, st) == F.ERR_INVALID_ARG
    assert fn(h, inp, 1, None, st) == F.ERR_INVALID_ARG
    assert fn(h, inp, 1, out, None) == F.ERR_INVALID_ARG
    assert lib.b200zk_last_error(h)
    assert fn(h, inp, 1, out, st) == 0 and (out.raw, st.raw[0]) == g.oracle(inp.raw)
    assert g.call(ctx, b"") == (b"", [])
    with pytest.raises(eb.B200Error):
        g.call(ctx, bytes(g.size + 1))
