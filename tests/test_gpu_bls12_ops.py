"""EIP-2537 G1/G2 addition and MSM on the device (b200zk_bls12_381_{g1,g2}_{add,msm}_batch): every output compared
byte-for-byte with the oracle's encoding (tests/bls12_ops_ref.py), closed forms on chain bases, scalar edge cases, every
status with neighbours intact, batches against single calls, the argument refusals, and the MSM tied to the pairing check
(which the reference's EIP-2537 vectors pin)."""
import ctypes as C

import numpy as np
import pytest

import bls12_ops_ref as ops
from bls12_ops_ref import G1, G2, P, R

pytestmark = pytest.mark.gpu

import ethrex_b200 as eb  # noqa: E402
from ethrex_b200 import _ffi as F  # noqa: E402

GROUPS = [G1, G2]


def _add(ctx, g, items):
    """items: [(a bytes, b bytes)] -> ([out per item], [status])"""
    fn = ctx.bls12_381_g1_add_batch if g is G1 else ctx.bls12_381_g2_add_batch
    out, st = fn(b"".join(a for a, _ in items), b"".join(b for _, b in items))
    return [out[g.size * i:g.size * (i + 1)] for i in range(len(items))], st


def _msm(ctx, g, calls):
    return (ctx.bls12_381_g1_msm_batch if g is G1 else ctx.bls12_381_g2_msm_batch)(calls)


def _expect(g, pt):
    return g.encode(pt), (1 if pt is None else 0)


def _off_subgroup(g, seed):
    return ops.G1_OFF_SUBGROUP if g is G1 and seed == 0 else g.random_point(2537 + seed)


# ---- malformed encodings (point -> bytes)
def _x_ge_p(g, pt):
    e = bytearray(g.encode(pt))
    e[16:64] = P.to_bytes(48, "big")
    return bytes(e)


def _y_ge_p(g, pt):
    e = bytearray(g.encode(pt))
    y = g.size // 2
    e[y + 16:y + 64] = (int.from_bytes(e[y + 16:y + 64], "big") + P).to_bytes(48, "big")
    return bytes(e)


def _last_ge_p(g, pt):  # G1: y, G2: y.c1 -- the last coordinate the loader reads
    e = bytearray(g.encode(pt))
    e[g.size - 48:] = (int.from_bytes(e[g.size - 48:], "big") + P).to_bytes(48, "big")
    return bytes(e)


def _padding(g, pt, byte=3):
    e = bytearray(g.encode(pt))
    e[g.size // 2 + byte] = 1
    return bytes(e)


def _off_curve(g, pt):
    x, y = pt
    return g.encode((x, (y + 1) % P) if g is G1 else (x, ((y[0] + 1) % P, y[1])))


# ---- addition ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g", GROUPS, ids=lambda g: g.name)
def test_add_group_law(ctx, g):
    p, q = g.mul(0x1234567, g.gen), g.mul(R - 0xABCDEF, g.gen)
    o1, o2 = _off_subgroup(g, 0), _off_subgroup(g, 1)
    assert not g.in_subgroup(o1) and not g.in_subgroup(o2)
    pairs = [(p, q), (p, p), (p, g.neg(p)), (None, p), (p, None), (None, None), (o1, o2), (o1, o1), (o2, g.neg(o2)), (o1, p)]
    outs, st = _add(ctx, g, [(g.encode(a), g.encode(b)) for a, b in pairs])
    for i, (a, b) in enumerate(pairs):
        assert (outs[i], st[i]) == _expect(g, g.add(a, b)), i
    assert st[2] == st[5] == st[8] == 1 and outs[2] == bytes(g.size)


@pytest.mark.parametrize("g", GROUPS, ids=lambda g: g.name)
def test_add_statuses_and_neighbours(ctx, g):
    p, q = g.mul(77, g.gen), g.mul(78, g.gen)
    good = (g.encode(p), g.encode(q))
    bad = [(_x_ge_p(g, p), 2), (_y_ge_p(g, p), 2), (_last_ge_p(g, p), 2), (_padding(g, p), 2), (_padding(g, p, 15), 2), (_off_curve(g, p), 3)]
    items, want = [], []
    for enc, s in bad:
        for side in range(2):
            items += [good, (enc, g.encode(q)) if side == 0 else (g.encode(q), enc)]
            want += [0, s]
    # 2 outranks 3 inside one item, whichever operand holds which
    items += [(_off_curve(g, p), _x_ge_p(g, q)), (_padding(g, q), _off_curve(g, p)), good]
    want += [2, 2, 0]
    outs, st = _add(ctx, g, items)
    assert st == want
    exp_good = g.encode(g.add(p, q))
    for o, s in zip(outs, st):
        assert o == (exp_good if s == 0 else bytes(g.size))


@pytest.mark.parametrize("g", GROUPS, ids=lambda g: g.name)
def test_add_batch_equals_single_calls(ctx, g):
    rng = np.random.default_rng(2537)
    pts = [g.mul(int(rng.integers(1, 1 << 62)), g.gen) for _ in range(6)] + [None, _off_subgroup(g, 0)]
    pool = [g.encode(x) for x in pts] + [_x_ge_p(g, pts[0]), _padding(g, pts[1]), _off_curve(g, pts[2])]
    items = [(pool[int(rng.integers(len(pool)))], pool[int(rng.integers(len(pool)))]) for _ in range(299)]
    items.insert(150, (g.encode(pts[0]), g.encode(g.neg(pts[0]))))  # at least one identity result
    outs, st = _add(ctx, g, items)
    for i, it in enumerate(items):
        o1, s1 = _add(ctx, g, [it])
        assert (outs[i], st[i]) == (o1[0], s1[0]), i
    assert set(st) == {0, 1, 2, 3}


# ---- MSM ----------------------------------------------------------------------------------------------------------------
A, D = 0x5EED, 0x1F1F1F


def _scalars(rng, n):
    return [int.from_bytes(rng.bytes(32), "big") for _ in range(n)]  # full 256-bit values, most of them >= r


@pytest.mark.parametrize("g", GROUPS, ids=lambda g: g.name)
def test_msm_chain_closed_forms(ctx, g):
    large = 4096 if g is G1 else 2048
    bases = g.chain(large, A, D)
    rng = np.random.default_rng(1109)
    sizes = [1, 2, 3, 64, large]
    ks = [_scalars(rng, k) for k in sizes]
    calls = [g.calldata(list(zip(bases[:k], s))) for k, s in zip(sizes, ks)]
    outs, st = _msm(ctx, g, calls)
    assert st == [0] * len(sizes)
    for k, s, o in zip(sizes, ks, outs):
        assert o == g.encode(g.chain_msm(s, A, D)), k


@pytest.mark.parametrize("g", GROUPS, ids=lambda g: g.name)
def test_msm_scalar_edges(ctx, g):
    q = g.mul(0xC0DE, g.gen)
    edges = [0, 1, R - 1, R, R + 1, (1 << 256) - 1, 2 * R, R - 2]
    calls = [g.calldata([(q, k)]) for k in edges] + [g.calldata([(q, k) for k in edges])]
    outs, st = _msm(ctx, g, calls)
    for i, k in enumerate(edges):
        assert (outs[i], st[i]) == _expect(g, g.mul(k % R, q)), hex(k)
    assert (outs[-1], st[-1]) == _expect(g, g.mul(sum(edges) % R, q))
    assert st[0] == st[3] == st[6] == 1


@pytest.mark.parametrize("g", GROUPS, ids=lambda g: g.name)
def test_msm_repeats_cancellation_identity_and_empty(ctx, g):
    q, q2 = g.mul(31337, g.gen), g.mul(4242, g.gen)
    k = 0x123456789ABCDEF
    cases = [[(q, 3), (q, 5)], [(q, k), (g.neg(q), k)], [(q, k), (q, R - k)], [(None, 5)], [(None, 5), (q, 2)],
             [(q, 1)] * 70 + [(q2, 2)] * 3, [(q, 1), (q, 1), (g.neg(q), 2)], []]
    outs, st = _msm(ctx, g, [g.calldata(c) for c in cases])
    for i, c in enumerate(cases):
        assert (outs[i], st[i]) == _expect(g, g.msm(c)), i
    assert st == [0, 1, 1, 1, 0, 0, 1, 1]


@pytest.mark.parametrize("g", GROUPS, ids=lambda g: g.name)
def test_msm_statuses_and_neighbours(ctx, g):
    q = g.mul(99, g.gen)
    off = _off_subgroup(g, 0)
    good = g.calldata([(q, 2), (g.gen, 3)])
    one = g.calldata([(q, 1)])
    pair = lambda enc, k=1: enc + k.to_bytes(32, "big")  # noqa: E731
    bad = [
        (pair(g.encode(off), 0), 3), (pair(g.encode(off), 1), 3), (one + pair(g.encode(off), 0), 3), (pair(g.encode(g.random_point(9))), 3),
        (pair(_off_curve(g, q)), 3), (pair(_x_ge_p(g, q)), 2), (pair(_y_ge_p(g, q)), 2), (pair(_padding(g, q)), 2),
        (one + pair(_last_ge_p(g, q), 0), 2),
        (pair(_off_curve(g, q)) + pair(_x_ge_p(g, q)), 2), (pair(_padding(g, q)) + pair(g.encode(off)), 2),
        (pair(g.encode(off)) + one * 100 + pair(_y_ge_p(g, q)), 2),
    ]
    calls, want = [], []
    for enc, s in bad:
        calls += [good, enc]
        want += [0, s]
    calls.append(good)
    want.append(0)
    outs, st = _msm(ctx, g, calls)
    assert st == want
    exp_good = g.encode(g.msm([(q, 2), (g.gen, 3)]))
    for o, s in zip(outs, st):
        assert o == (exp_good if s == 0 else bytes(g.size))


@pytest.mark.parametrize("g", GROUPS, ids=lambda g: g.name)
def test_msm_batch_equals_single_calls(ctx, g):
    bases = g.chain(300, A, D)
    rng = np.random.default_rng(1246)
    calls, good = [], []
    for k in (0, 1, 17, 300, 5, 0, 64, 2, 17, 1, 40):
        s = _scalars(rng, k)
        calls.append(g.calldata(list(zip(bases[:k], s))))
        good.append(g.encode(g.chain_msm(s, A, D)))
    for i, (enc, bad_pt) in enumerate(((2, _off_curve(g, bases[5])), (4, _x_ge_p(g, bases[1])), (8, g.encode(_off_subgroup(g, 0))))):
        c = bytearray(calls[enc])
        j = g.pair * (3 + i)
        c[j:j + g.size] = bad_pt
        calls[enc] = bytes(c)
    outs, st = _msm(ctx, g, calls)
    assert st == [1, 0, 3, 0, 2, 1, 0, 0, 3, 0, 0]
    for i, c in enumerate(calls):
        o1, s1 = _msm(ctx, g, [c])
        assert (outs[i], st[i]) == (o1[0], s1[0]), i
        if st[i] == 0:
            assert outs[i] == good[i], i


def test_msm_tied_to_the_pairing(ctx):
    """e(sum k_i P_i, -G2) prod e(P_i, [k_i] G2) = 1 and e(-G1, sum k_i Q_i) prod e([k_i] G1, Q_i) = 1 on the device's
    pairing check, which the reference's EIP-2537 vectors pin"""
    import bls_pairing_ref as B
    rng = np.random.default_rng(2539)
    ks = [int(rng.integers(1, 1 << 62)) for _ in range(4)]
    ps = [G1.mul(int(rng.integers(1, 1 << 62)), G1.gen) for _ in ks]
    qs = [G2.mul(int(rng.integers(1, 1 << 62)), G2.gen) for _ in ks]
    (m1,), st1 = _msm(ctx, G1, [G1.calldata(list(zip(ps, ks)))])
    (m2,), st2 = _msm(ctx, G2, [G2.calldata(list(zip(qs, ks)))])
    assert st1 == st2 == [0]
    check1 = m1 + B.g2_eip2537(B.g2_neg(B.G2)) + b"".join(B.g1_eip2537(p) + B.g2_eip2537(B.g2_mul(k, B.G2)) for p, k in zip(ps, ks))
    check2 = B.g1_eip2537(G1.neg(B.G1)) + m2 + b"".join(B.g1_eip2537(G1.mul(k, B.G1)) + B.g2_eip2537(q) for q, k in zip(qs, ks))
    wrong = G1.encode(G1.add(B.g1_from_eip2537(m1), G1.gen)) + check1[128:]
    res, st = ctx.bls12_381_pairing_check_batch([check1, check2, wrong])
    assert (res, st) == ([1, 1, 0], [0, 0, 0])


@pytest.mark.parametrize("g", GROUPS, ids=lambda g: g.name)
def test_refusals(ctx, g):
    lib, h = F.lib, ctx._h
    add = lib.b200zk_bls12_381_g1_add_batch if g is G1 else lib.b200zk_bls12_381_g2_add_batch
    msm = lib.b200zk_bls12_381_g1_msm_batch if g is G1 else lib.b200zk_bls12_381_g2_msm_batch
    pt = C.create_string_buffer(g.calldata([(g.gen, 1)]), g.pair)
    out, st = C.create_string_buffer(2 * g.size), C.create_string_buffer(2)

    def offs(*v):
        return (C.c_uint32 * len(v))(*v)
    assert add(h, None, None, 0, None, None) == 0
    assert msm(h, None, None, 0, None, None) == 0
    assert add(h, None, pt, 1, out, st) == F.ERR_INVALID_ARG
    assert add(h, pt, pt, 1, None, st) == F.ERR_INVALID_ARG
    assert add(h, pt, pt, 1, out, None) == F.ERR_INVALID_ARG
    assert lib.b200zk_last_error(h)
    assert msm(h, None, offs(0, 1), 1, out, st) == F.ERR_INVALID_ARG
    assert msm(h, pt, None, 1, out, st) == F.ERR_INVALID_ARG
    assert msm(h, pt, offs(0, 1), 1, None, st) == F.ERR_INVALID_ARG
    assert msm(h, pt, offs(1, 1), 1, out, st) == F.ERR_INVALID_ARG
    assert b"pair_offsets[0]" in lib.b200zk_last_error(h)
    assert msm(h, pt, offs(0, 1, 0), 2, out, st) == F.ERR_INVALID_ARG
    assert b"non-decreasing" in lib.b200zk_last_error(h)
    assert msm(h, None, offs(0, 0), 1, out, st) == 0 and st.raw[0] == 1 and out.raw[:g.size] == bytes(g.size)  # empty call
    assert msm(h, pt, offs(0, 1), 1, out, st) == 0 and st.raw[0] == 0 and out.raw[:g.size] == g.encode(g.gen)
    with pytest.raises(eb.B200Error):
        (ctx.bls12_381_g1_add_batch if g is G1 else ctx.bls12_381_g2_add_batch)(bytes(g.size), bytes(g.size + 1))
    with pytest.raises(eb.B200Error):
        _msm(ctx, g, [bytes(g.pair - 1)])
