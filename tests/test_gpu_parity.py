"""GPU parity tests: libb200zk.so (through the C ABI) against the CPU oracle, bit exact.

Mirrors the shape of the reference's precompile KAT tests
(/root/reference/test/tests/levm/precompile_tests.rs:6-151: feed bytes, compare bytes, check the error
variant) for the operations of SURVEY.md section 8a rows a6-a8.
"""
import os

import numpy as np
import pytest

import cpu_oracle as orc
import pyref
from helpers import (chain_kd, dev_empty, expected_chain_msm_g1, expected_chain_msm_g2, scalars_special, to_dev,
                     to_host)

pytestmark = pytest.mark.gpu

import ethrex_b200 as eb  # noqa: E402


# ------------------------------------------------------------------------------------------ field core
@pytest.mark.parametrize("which,field", [(0, "fq"), (1, "fr")])
def test_field_mul_matches_oracle(ctx, which, field):
    n = 4096
    mod = pyref.P if which == 0 else pyref.R
    rng = np.random.default_rng(1234 + which)
    vals_a = [int.from_bytes(rng.bytes(32), "little") % mod for _ in range(n)]
    vals_b = [int.from_bytes(rng.bytes(32), "little") % mod for _ in range(n)]
    # edge values: 0, 1, p-1, R mod p ...
    edge = [0, 1, mod - 1, mod - 2, (1 << 256) % mod, 2, (1 << 253) % mod]
    for i, e in enumerate(edge):
        vals_a[i] = e
        vals_b[-1 - i] = e
        vals_b[i] = edge[(i * 3) % len(edge)]
    a, b = orc.ints_to_array(vals_a), orc.ints_to_array(vals_b)
    da, db, do = to_dev(a), to_dev(b), dev_empty(4 * n)
    ctx.field_mul_device(da, db, do, n, which)
    got = to_host(do).reshape(n, 4)
    assert (got == orc.field_mul(field, a, b)).all()
    # chained products (the throughput path) == repeated oracle products
    ctx.field_mul_device(da, db, do, n, which, repeat=5)
    exp = a
    for _ in range(5):
        exp = orc.field_mul(field, exp, b)
    assert (to_host(do).reshape(n, 4) == exp).all()
    # the dedicated squaring (36 instead of 64 products) against the oracle's a*a, once and chained; extra edge
    # values exercise every limb's top bit (the doubled multiplicand) and the all-ones patterns
    more = [(mod - 1) >> 1, ((1 << 254) - 1) % mod, 0x80000000, (0x80000000 << 32) | 0x80000000, sum(0x80000000 << (32 * k) for k in range(8)) % mod,
            sum(0xffffffff << (32 * k) for k in range(7)), (mod >> 1) + 1]
    for i, e in enumerate(more):
        vals_a[len(edge) + i] = e % mod
    a = orc.ints_to_array(vals_a)
    da = to_dev(a)
    ctx.field_mul_device(da, db, do, n, which + 2)
    assert (to_host(do).reshape(n, 4) == orc.field_mul(field, a, a)).all()
    ctx.field_mul_device(da, db, do, n, which + 2, repeat=4)
    exp = a
    for _ in range(4):
        exp = orc.field_mul(field, exp, exp)
    assert (to_host(do).reshape(n, 4) == exp).all()


def test_mont_roundtrip_and_random(ctx):
    n = 5000
    d = dev_empty(4 * n)
    ctx.fr_random_device(d, n, pyref.SEED_SCALARS, 0)
    host = to_host(d).reshape(n, 4)
    assert (host == orc.rand_fr(pyref.SEED_SCALARS, 0, n)).all()
    ctx.field_to_mont_device(d, n, 1)
    assert (to_host(d).reshape(n, 4) == orc.fr_to_mont(host)).all()
    ctx.field_from_mont_device(d, n, 1)
    assert (to_host(d).reshape(n, 4) == host).all()
    ctx.fr_random_device(d, n, pyref.SEED_NTT, 77, eb.SCALARS_MONT)
    assert (to_host(d).reshape(n, 4) == orc.fr_to_mont(orc.rand_fr(pyref.SEED_NTT, 77, n))).all()
    # Fq (which = 0): random values and the edges 0, 1, p - 1, p, 2^256 - 1 (to_mont reduces its input first)
    rng = np.random.default_rng(0xF9)
    vals = [int.from_bytes(rng.bytes(32), "little") % pyref.P for _ in range(n)]
    edges = [0, 1, pyref.P - 1, pyref.P, pyref.P + 1, (1 << 256) - 1, (1 << 255), (1 << 254) - 1]
    vals[:len(edges)] = edges
    canon = orc.ints_to_array([v % pyref.P for v in vals])
    d = to_dev(orc.ints_to_array(vals))
    ctx.field_to_mont_device(d, n, 0)
    mont = orc.fq_to_mont(canon)
    assert (to_host(d).reshape(n, 4) == mont).all()
    assert orc.array_to_ints(mont[:3]) == [0, (1 << 256) % pyref.P, (pyref.P - 1) * (1 << 256) % pyref.P]
    ctx.field_from_mont_device(d, n, 0)
    assert (to_host(d).reshape(n, 4) == canon).all()


@pytest.mark.parametrize("n", [1, 255, 256, 257, 33 * 4096 + 1, 1 << 20])
def test_fr_quotient_matches_oracle(ctx, n):
    """fr_quotient_device, the pointwise step (a*b - c) * zinv of the Groth16 quotient, against the oracle: rows holding
    0, 1 and r - 1 in every operand, zinv in {1, r - 1, random}, into a separate buffer and in place over a (how
    ethrex_b200/groth16.py calls it)"""
    a, b, c = (orc.rand_fr(0xF0 + j, 0, n) for j in range(3))
    edges = [0, 1, pyref.R - 1]
    for row in range(min(n, 9)):
        a[row] = orc.int_to_limbs(edges[row % 3])
        b[row] = orc.int_to_limbs(edges[(row // 3) % 3])
        c[row] = orc.int_to_limbs(edges[(row + 1) % 3])
    a, b, c = orc.fr_to_mont(a), orc.fr_to_mont(b), orc.fr_to_mont(c)
    da, db, dc = to_dev(a), to_dev(b), to_dev(c)
    for zinv in (1, pyref.R - 1, pyref.rand_fr(0xF3, n)):
        exp = orc.fr_quotient(a, b, c, zinv)
        out = dev_empty(4 * n)
        ctx.fr_quotient_device(da, db, dc, out, n, zinv)
        assert (to_host(out).reshape(n, 4) == exp).all(), zinv
        inplace = da.clone()
        ctx.fr_quotient_device(inplace, db, dc, inplace, n, zinv)
        assert (to_host(inplace).reshape(n, 4) == exp).all(), zinv


# ------------------------------------------------------------------------------------------ synthetic bases
def test_chain_generators_match_oracle(ctx):
    k, d = chain_kd()
    n = 300
    g1 = dev_empty(8 * n)
    ctx.g1_chain_device(g1, 5, n, k, d)
    assert (to_host(g1).reshape(n, 8) == orc.g1_chain(n + 5, k, d)[5:]).all()
    assert ctx.g1_check_device(g1, n) == n
    g2 = dev_empty(16 * n)
    ctx.g2_chain_device(g2, 0, n, k, d)
    assert (to_host(g2).reshape(n, 16) == orc.g2_chain(n, k, d)).all()
    assert ctx.g2_check_device(g2, n) == n
    # corrupt one point: the checker must name it
    h = to_host(g1).copy().reshape(n, 8)
    h[123, 0] ^= 1
    assert ctx.g1_check_device(to_dev(h), n) == 123


# ------------------------------------------------------------------------------------------ NTT
def _ntt_case(ctx, log_n, flags, coset_gen=None, seed=pyref.SEED_NTT):
    n = 1 << log_n
    a = orc.fr_to_mont(orc.rand_fr(seed, 0, n))
    d = to_dev(a)
    oflags = (orc.NTT_INVERSE if flags & eb.NTT_INVERSE else 0) | (orc.NTT_COSET if flags & eb.NTT_COSET else 0)
    ctx.fr_ntt_device(d, log_n, flags, None if coset_gen is None else coset_gen.to_bytes(32, "little"))
    exp = orc.fr_ntt(a, log_n, oflags, coset_gen=coset_gen)
    got = to_host(d).reshape(n, 4)
    assert (got == exp).all(), f"log_n={log_n} flags={flags}"


@pytest.mark.parametrize("log_n", list(range(0, 15)))
def test_ntt_small_all_modes(ctx, log_n):
    for flags in (0, eb.NTT_INVERSE, eb.NTT_COSET, eb.NTT_INVERSE | eb.NTT_COSET):
        _ntt_case(ctx, log_n, flags)
    _ntt_case(ctx, log_n, eb.NTT_COSET, coset_gen=7)
    _ntt_case(ctx, log_n, eb.NTT_COSET | eb.NTT_INVERSE, coset_gen=pyref.R - 3)


@pytest.mark.parametrize("log_n", [16, 17, 20, 22])
def test_ntt_medium_vs_oracle(ctx, log_n):
    _ntt_case(ctx, log_n, 0)
    _ntt_case(ctx, log_n, eb.NTT_INVERSE)


@pytest.mark.parametrize("log_n", [17, 18, 21])
def test_ntt_direct_twiddle_table_all_modes(ctx, log_n, monkeypatch):
    """Sizes above 2^16 take the last pass's inter-pass twiddles from a direct N-entry table (one lookup, one product), built
    on first use per (direction, scaled); B200ZK_NTT_FULL_TW=0 keeps the two-level tables.  Both must be the oracle's bytes in
    every mode (the plain inverse folds n^-1 into the table, the coset inverse must not)."""
    modes = [(0, None), (eb.NTT_INVERSE, None), (eb.NTT_COSET, None), (eb.NTT_INVERSE | eb.NTT_COSET, None), (eb.NTT_COSET, 7), (eb.NTT_COSET | eb.NTT_INVERSE, pyref.R - 3)]
    for knob in ("26", "0"):
        monkeypatch.setenv("B200ZK_NTT_FULL_TW", knob)
        for flags, gen in modes:
            _ntt_case(ctx, log_n, flags, coset_gen=gen)


def test_ntt_golden_2_12(ctx):
    """config #1: 2^12 forward against the pure-Python fixture (tests/golden/ntt_2_12.npz)."""
    import os
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "ntt_2_12.npz"))
    a = g["input_canonical"]
    d = to_dev(a)
    ctx.fr_ntt_device(d, 12, eb.NTT_CANONICAL)
    assert (to_host(d).reshape(-1, 4) == g["forward_canonical"]).all()
    ctx.fr_ntt_device(d, 12, eb.NTT_CANONICAL | eb.NTT_INVERSE)
    assert (to_host(d).reshape(-1, 4) == a).all()


def test_ntt_special_inputs(ctx):
    log_n, n = 10, 1024
    one_m = orc.fr_to_mont(orc.ints_to_array([1]))[0]
    # delta at 0 -> all ones ; all ones -> n * delta
    delta = np.zeros((n, 4), dtype=np.uint64)
    delta[0] = one_m
    d = to_dev(delta)
    ctx.fr_ntt_device(d, log_n, 0)
    assert (to_host(d).reshape(n, 4) == np.tile(one_m, (n, 1))).all()
    ctx.fr_ntt_device(d, log_n, 0)
    got = orc.array_to_ints(orc.fr_from_mont(to_host(d).reshape(n, 4)))
    assert got[0] == n and all(v == 0 for v in got[1:])
    # a[j] = j (canonical in/out path, big-endian flavour too)
    ramp = orc.ints_to_array(list(range(n)))
    d = to_dev(ramp)
    ctx.fr_ntt_device(d, log_n, eb.NTT_CANONICAL)
    assert orc.array_to_ints(to_host(d)) == pyref.ntt_fast(list(range(n)))
    be = b"".join(pyref.fr_to_be(v) for v in range(n))
    dbe = to_dev(np.frombuffer(be, dtype=np.uint64))
    ctx.fr_ntt_device(dbe, log_n, eb.NTT_BE)
    exp_be = b"".join(pyref.fr_to_be(v) for v in pyref.ntt_fast(list(range(n))))
    assert to_host(dbe).tobytes() == exp_be


def test_ntt_host_entry_point(ctx):
    log_n, n = 13, 1 << 13
    a = orc.fr_to_mont(orc.rand_fr(99, 0, n))
    buf = a.copy()
    ctx.fr_ntt(buf, log_n, 0)
    assert (buf == orc.fr_ntt(a, log_n)).all()
    ctx.fr_ntt(buf, log_n, eb.NTT_INVERSE)
    assert (buf == a).all()


def test_ntt_2_24_roundtrip_and_spot_check(ctx):
    """config #3 at full size: iNTT(NTT(a)) == a, linearity probe, and direct evaluation of a few outputs."""
    import torch
    log_n, n = 24, 1 << 24
    d = dev_empty(4 * n)
    ctx.fr_random_device(d, n, pyref.SEED_NTT, 0, eb.SCALARS_MONT)
    orig = d.clone()
    ctx.fr_ntt_device(d, log_n, 0)
    fwd = d.clone()
    ctx.fr_ntt_device(d, log_n, eb.NTT_INVERSE)
    assert torch.equal(d, orig)
    # full compare against the CPU oracle's transform
    exp = orc.fr_ntt(to_host(orig).reshape(n, 4), log_n)
    assert (to_host(fwd).reshape(n, 4) == exp).all()


# ------------------------------------------------------------------------------------------ MSM
def _msm_g1_vs_oracle(ctx, n, scalars, method=0):
    k, d = chain_kd()
    pts = orc.g1_chain(max(n, 1), k, d)[:n]
    got = ctx.g1_msm_device(to_dev(pts) if n else dev_empty(8), to_dev(scalars) if n else dev_empty(4), n)
    assert got == orc.g1_msm(pts, scalars, method), f"n={n}"
    return got


@pytest.mark.parametrize("n", [0, 1, 2, 3, 31, 32, 33, 100, 1000, 4096])
def test_g1_msm_small_vs_oracle(ctx, n):
    _msm_g1_vs_oracle(ctx, n, scalars_special(n) if n else np.zeros((0, 4), dtype=np.uint64))


def test_g1_msm_kats_from_reference(ctx):
    """n=1 MSMs reproduce the reference's own scalar-multiplication KATs (SURVEY.md section 8):
    7*(1,2) (test/tests/l2/integration_tests.rs:572) and 2*(1,2)."""
    g = orc.g1_be_to_native(pyref.g1_to_be(pyref.G1_GEN))
    for s, exp in ((7, "17072b2ed3bb8d759a5325f477629386cb6fc6ecb801bd76983a6b86abffe078168ada6cd130dd52017bb54bfa19377aadfe3bf05d18f41b77809f7f60d4af9e"),
                   (2, "030644e72e131a029b85045b68181585d97816a916871ca8d3c208c16d87cfd315ed738c0e0a7c92e7845f96b2ae9c0a68a6a449e3538fc7ff3ebf7a5a18a2c4")):
        got = ctx.g1_msm_device(to_dev(g), to_dev(orc.ints_to_array([s])), 1)
        assert got.hex() == exp
    # r*G = identity -> (0,0) and status OK_INFINITY is folded into the bytes
    assert ctx.g1_msm_device(to_dev(g), to_dev(orc.ints_to_array([pyref.R])), 1) == bytes(64)


def _group(g2):
    """(chain, device MSM, oracle MSM, native -> BE) of G1 or G2"""
    return ((orc.g2_chain, "g2_msm_device", orc.g2_msm, orc.g2_native_to_be) if g2 else
            (orc.g1_chain, "g1_msm_device", orc.g1_msm, orc.g1_native_to_be))


def _negate_native(pts_row, g2):
    """-P of one native point: y -> p - y coordinate-wise (BE: G1 x|y, G2 x_im|x_re|y_im|y_re)"""
    size = 128 if g2 else 64
    raw = bytearray((orc.g2_native_to_be if g2 else orc.g1_native_to_be)(np.ascontiguousarray(pts_row)))
    for off in ((64, 96) if g2 else (32,)):
        raw[off:off + 32] = ((pyref.P - int.from_bytes(raw[off:off + 32], "big")) % pyref.P).to_bytes(32, "big")
    return (orc.g2_be_to_native if g2 else orc.g1_be_to_native)(bytes(raw[:size]))[0]


def _msm_edge_distributions(ctx, g2):
    chain, dev_msm, oracle_msm, _ = _group(g2)
    msm = getattr(ctx, dev_msm)
    k, d = chain_kd()
    n = 2048
    pts = chain(n, k, d)
    dp = to_dev(pts)
    cases = {
        "all_zero": [0] * n,
        "all_one": [1] * n,
        "all_r_minus_1": [pyref.R - 1] * n,
        "small": [(i * 2654435761) & 0xFFFF for i in range(n)],
        "half_zero": [0 if i & 1 else pyref.rand_fr(5, i) for i in range(n)],
        "unreduced": [pyref.R + 5 + i for i in range(n)],          # >= r: reduced mod r by the library
        "max_u256": [(1 << 256) - 1 - i for i in range(n)],
    }
    for name, vals in cases.items():
        s = orc.ints_to_array(vals)
        assert msm(dp, to_dev(s), n) == oracle_msm(pts, s), name
    # repeated points, P and -P pairs, identity points among the bases
    pts2 = pts.copy()
    pts2[1] = pts2[0]
    pts2[3] = pts2[2]
    pts2[5] = _negate_native(pts[4:5], g2)
    pts2[7] = 0
    s = orc.rand_fr(11, 0, n)
    s[1] = s[0]
    s[5] = s[4]
    s[3] = orc.int_to_limbs((pyref.R - orc.limbs_to_int(s[2])) % pyref.R)
    assert msm(to_dev(pts2), to_dev(s), n) == oracle_msm(pts2, s)


def test_g1_msm_edge_distributions(ctx):
    _msm_edge_distributions(ctx, g2=False)


def test_g2_msm_edge_distributions(ctx):
    _msm_edge_distributions(ctx, g2=True)


def _msm_window_sweep(ctx, g2):
    chain, dev_msm, oracle_msm, _ = _group(g2)
    k, d = chain_kd()
    n = 3000
    pts, s = chain(n, k, d), scalars_special(n)
    exp = oracle_msm(pts, s)
    dp, ds = to_dev(pts), to_dev(s)
    try:
        for c in (2, 3, 5, 8, 11, 13, 16):
            ctx.set_msm_window(c)
            assert getattr(ctx, dev_msm)(dp, ds, n) == exp, f"c={c}"
    finally:
        ctx.set_msm_window(0)


def test_g1_msm_window_sweep(ctx):
    _msm_window_sweep(ctx, g2=False)


def test_g2_msm_window_sweep(ctx):
    _msm_window_sweep(ctx, g2=True)


def _msm_scalar_formats(ctx, g2):
    chain, dev_msm, oracle_msm, native_to_be = _group(g2)
    msm = getattr(ctx, dev_msm)
    k, d = chain_kd()
    n = 777
    pts, s = chain(n, k, d), scalars_special(n)
    exp = oracle_msm(pts, s)
    dp = to_dev(pts)
    assert msm(dp, to_dev(orc.fr_to_mont(s)), n, eb.SCALARS_MONT) == exp
    be = b"".join(pyref.fr_to_be(v) for v in orc.array_to_ints(s))
    assert msm(dp, to_dev(np.frombuffer(be, dtype=np.uint64)), n, eb.SCALARS_BE) == exp
    native = msm(dp, to_dev(s), n, eb.OUT_NATIVE)
    assert native_to_be(np.frombuffer(native, dtype=np.uint64)) == exp


def test_g1_msm_scalar_formats(ctx):
    _msm_scalar_formats(ctx, g2=False)


def test_g2_msm_scalar_formats(ctx):
    _msm_scalar_formats(ctx, g2=True)


@pytest.mark.parametrize("log_n", [16, 20])
def test_g1_msm_large_closed_form(ctx, log_n):
    """config #2 (2^20): synthetic chain bases make the exact result a single scalar multiplication."""
    n = 1 << log_n
    k, d = chain_kd()
    dp, ds = dev_empty(8 * n), dev_empty(4 * n)
    ctx.g1_chain_device(dp, 0, n, k, d)
    ctx.fr_random_device(ds, n, pyref.SEED_SCALARS, 0)
    got = ctx.g1_msm_device(dp, ds, n)
    s = to_host(ds).reshape(n, 4)
    assert got == expected_chain_msm_g1(s, k, d)
    if log_n == 16:
        assert got == orc.g1_msm(to_host(dp).reshape(n, 8), s)


def test_g1_msm_2_24_closed_form(ctx):
    n = 1 << 24
    k, d = chain_kd()
    dp, ds = dev_empty(8 * n), dev_empty(4 * n)
    ctx.g1_chain_device(dp, 0, n, k, d)
    assert ctx.g1_check_device(dp, n) == n
    ctx.fr_random_device(ds, n, pyref.SEED_SCALARS, 0)
    got = ctx.g1_msm_device(dp, ds, n)
    assert got == expected_chain_msm_g1(to_host(ds).reshape(n, 4), k, d)


@pytest.mark.parametrize("n", [0, 1, 2, 33, 500, 4096])
def test_g2_msm_small_vs_oracle(ctx, n):
    k, d = chain_kd()
    pts = orc.g2_chain(max(n, 1), k, d)[:n]
    s = scalars_special(n) if n else np.zeros((0, 4), dtype=np.uint64)
    got = ctx.g2_msm_device(to_dev(pts) if n else dev_empty(16), to_dev(s) if n else dev_empty(4), n)
    assert got == orc.g2_msm(pts, s)


def test_g2_msm_2_18_closed_form(ctx):
    n = 1 << 18
    k, d = chain_kd()
    dp, ds = dev_empty(16 * n), dev_empty(4 * n)
    ctx.g2_chain_device(dp, 0, n, k, d)
    ctx.fr_random_device(ds, n, pyref.SEED_SCALARS, 0)
    assert ctx.g2_msm_device(dp, ds, n) == expected_chain_msm_g2(to_host(ds).reshape(n, 4), k, d)


# ------------------------------------------------------------------------------------------ host entry points, errors
def test_host_msm_be_and_native(ctx):
    k, d = chain_kd()
    n = 600
    pts, s = orc.g1_chain(n, k, d), scalars_special(n)
    exp = orc.g1_msm(pts, s)
    assert ctx.g1_msm(pts, s, n) == exp
    be_pts = orc.g1_native_to_be(pts)
    be_s = b"".join(pyref.fr_to_be(v) for v in orc.array_to_ints(s))
    assert ctx.g1_msm(be_pts, be_s, n, eb.POINTS_BE | eb.SCALARS_BE) == exp
    pts2 = orc.g2_chain(n, k, d)
    exp2 = orc.g2_msm(pts2, s)
    assert ctx.g2_msm(pts2, s, n) == exp2
    assert ctx.g2_msm(orc.g2_native_to_be(pts2), be_s, n, eb.POINTS_BE | eb.SCALARS_BE) == exp2


def test_host_msm_rejects_bad_points(ctx):
    """error behaviour of provider.rs:217-219 / precompiles.rs:801-820: not on curve, coordinate >= p."""
    g = pyref.g1_to_be(pyref.G1_GEN)
    s = (5).to_bytes(32, "big")
    bad_curve = (1).to_bytes(32, "big") + (3).to_bytes(32, "big")
    with pytest.raises(eb.B200Error) as e:
        ctx.g1_msm(g + bad_curve, s + s, 2, eb.POINTS_BE | eb.SCALARS_BE)
    assert e.value.status == 3 and e.value.kind == "Serialization"
    # the out-of-range x of precompile_tests.rs:143-151 (p+1, p+2)
    oob = (pyref.P + 1).to_bytes(32, "big") + (pyref.P + 2).to_bytes(32, "big")
    with pytest.raises(eb.B200Error) as e:
        ctx.g1_msm(oob + g, s + s, 2, eb.POINTS_BE | eb.SCALARS_BE)
    assert e.value.status == 2
    # identity encodes as (0,0) and is accepted
    assert ctx.g1_msm(bytes(64) + g, s + s, 2, eb.POINTS_BE | eb.SCALARS_BE) == pyref.g1_to_be(pyref.g1_mul(5, pyref.G1_GEN))


def test_resident_bases(ctx):
    k, d = chain_kd()
    n = 5000
    pts = orc.g1_chain(n, k, d)
    h = ctx.g1_bases_upload(pts, n)
    try:
        for m in (n, 1234, 1):
            s = orc.rand_fr(m, 0, m)
            assert ctx.g1_msm_resident(h, s, m) == orc.g1_msm(pts[:m], s)
        with pytest.raises(eb.B200Error):
            ctx.g1_msm_resident(h, orc.rand_fr(1, 0, n + 1), n + 1)
        with pytest.raises(eb.B200Error):
            ctx.g2_msm_resident(h, orc.rand_fr(1, 0, 4), 4)
    finally:
        ctx.bases_free(h)
    pts2 = orc.g2_chain(300, k, d)
    h2 = ctx.g2_bases_upload(orc.g2_native_to_be(pts2), 300, eb.POINTS_BE)
    s = orc.rand_fr(3, 0, 300)
    assert ctx.g2_msm_resident(h2, s, 300) == orc.g2_msm(pts2, s)
    ctx.bases_free(h2)


def test_partials_fold_equals_whole(ctx):
    """the multi-GPU combine on one device: MSM(shard0) + MSM(shard1) + ... == MSM(all)."""
    import torch
    k, d = chain_kd()
    n, shards = 6000, 4
    pts, s = orc.g1_chain(n, k, d), orc.rand_fr(21, 0, n)
    parts = torch.zeros(shards * 16, dtype=torch.int64, device="cuda")
    per = n // shards
    for r in range(shards):
        ctx.g1_msm_partial_device(to_dev(pts[r * per:(r + 1) * per]), to_dev(s[r * per:(r + 1) * per]), per, parts[r * 16:(r + 1) * 16])
    assert ctx.g1_fold_partials_device(parts, shards) == orc.g1_msm(pts, s)
    pts2 = orc.g2_chain(1000, k, d)
    parts2 = torch.zeros(2 * 32, dtype=torch.int64, device="cuda")
    ctx.g2_msm_partial_device(to_dev(pts2[:500]), to_dev(s[:500]), 500, parts2[:32])
    ctx.g2_msm_partial_device(to_dev(pts2[500:]), to_dev(s[500:1000]), 500, parts2[32:])
    assert ctx.g2_fold_partials_device(parts2, 2) == orc.g2_msm(pts2, s[:1000])


def test_launch_counter_moves(ctx):
    before = ctx.launch_count
    d = dev_empty(4 * 16)
    ctx.fr_random_device(d, 16, 1, 0)
    assert ctx.launch_count == before + 1


def test_precomputed_window_tables(ctx):
    """resident bases expanded to 2^(c*w)*P_i: same group element, for full and partial use of the table."""
    k, d = chain_kd()
    n = 3000
    pts = orc.g1_chain(n, k, d)
    for c in (0, 5, 9, 13):
        h = ctx.g1_bases_upload(pts, n)
        ctx.bases_precompute(h, c)
        try:
            for m in (n, 777, 1):
                s = scalars_special(m, seed=400 + m)
                exp = orc.g1_msm(pts[:m], s)
                assert ctx.g1_msm_resident(h, s, m) == exp, (c, m)
                assert ctx.g1_msm_resident_device(h, to_dev(s), m) == exp, (c, m)
            with pytest.raises(eb.B200Error):
                ctx.bases_precompute(h, 0)  # already a table
        finally:
            ctx.bases_free(h)
    # from device memory, G2, and edge distributions
    dp = to_dev(pts)
    h = ctx.g1_bases_from_device(dp, n)
    ctx.bases_precompute(h, 11)
    for vals in ([0] * n, [1] * n, [pyref.R - 1] * n, [(1 << 256) - 1 - i for i in range(n)]):
        s = orc.ints_to_array(vals)
        assert ctx.g1_msm_resident_device(h, to_dev(s), n) == orc.g1_msm(pts, s)
    ctx.bases_free(h)
    pts2 = orc.g2_chain(600, k, d)
    h2 = ctx.g2_bases_from_device(to_dev(pts2), 600)
    ctx.bases_precompute(h2, 0)
    s = scalars_special(600, seed=9)
    assert ctx.g2_msm_resident_device(h2, to_dev(s), 600) == orc.g2_msm(pts2, s)
    assert ctx.g2_msm_resident(h2, s[:100], 100) == orc.g2_msm(pts2[:100], s[:100])
    ctx.bases_free(h2)


def test_precomputed_2_20_closed_form(ctx):
    n = 1 << 20
    k, d = chain_kd()
    dp, ds = dev_empty(8 * n), dev_empty(4 * n)
    ctx.g1_chain_device(dp, 0, n, k, d)
    ctx.fr_random_device(ds, n, pyref.SEED_SCALARS, 0)
    h = ctx.g1_bases_from_device(dp, n)
    ctx.bases_precompute(h, 0)
    try:
        assert ctx.g1_msm_resident_device(h, ds, n) == expected_chain_msm_g1(to_host(ds).reshape(n, 4), k, d)
    finally:
        ctx.bases_free(h)


def test_pair_sum_rounds_edge_cases(ctx):
    """batched-affine pre-pass: equal points (tangent), opposite points (identity), identity operands, heavy buckets."""
    k, d = chain_kd()
    n = 4096
    pts = orc.g1_chain(n, k, d)
    pts[1] = pts[0]; pts[3] = pts[2]; pts[9] = pts[8]                       # repeated bases
    neg = orc.g1_be_to_native(pyref.g1_to_be(pyref.pt_neg(pyref._Fq, pyref.g1_from_be(orc.g1_native_to_be(pts[4:5])))))
    pts[5] = neg[0]                                                          # P and -P
    pts[7] = 0; pts[11] = 0                                                  # identity bases
    cases = {
        "random": scalars_special(n),
        "all_one": orc.ints_to_array([1] * n),                               # one heavy bucket, every pair in it
        "all_same": orc.ints_to_array([0x1234567] * n),
        "pairs": orc.ints_to_array([(i // 2) * 7919 + 1 for i in range(n)]),  # neighbours share their digits
    }
    dp = to_dev(pts)
    try:
        for c in (6, 11):
            ctx.set_msm_window(c)
            for rounds in (1, 2, 3, 4):
                ctx.set_msm_pair_rounds(rounds)
                for name, s in cases.items():
                    assert ctx.g1_msm_device(dp, to_dev(s), n) == orc.g1_msm(pts, s), (c, rounds, name)
        ctx.set_msm_window(0)
        pts2 = orc.g2_chain(512, k, d)
        pts2[1] = pts2[0]
        s2 = orc.ints_to_array([3] * 512)
        for rounds in (1, 3):
            ctx.set_msm_pair_rounds(rounds)
            assert ctx.g2_msm_device(to_dev(pts2), to_dev(s2), 512) == orc.g2_msm(pts2, s2)
    finally:
        ctx.set_msm_window(0)
        ctx.set_msm_pair_rounds(-1)


def test_pipelined_chunks_match(ctx):
    """chunk-pipelined schedule (sort of chunk k+1 overlapping the accumulation of chunk k): same bytes as one shot."""
    k, d = chain_kd()
    n = 10007
    pts, s = orc.g1_chain(n, k, d), scalars_special(n)
    exp = orc.g1_msm(pts, s)
    dp, ds = to_dev(pts), to_dev(s)
    h = ctx.g1_bases_upload(pts, n)
    ht = ctx.g1_bases_upload(pts, n)
    ctx.bases_precompute(ht, 9)
    try:
        for chunks in (1, 2, 3, 7, 40):
            ctx.set_msm_chunks(chunks)
            assert ctx.g1_msm_device(dp, ds, n) == exp, chunks
            assert ctx.g1_msm_resident(h, s, n) == exp, chunks            # host scalars: upload rides in the pipeline
            assert ctx.g1_msm_resident_device(ht, ds, n) == exp, chunks    # merged table, chunk offsets into it
            assert ctx.g1_msm_resident(ht, s[:5000], 5000) == orc.g1_msm(pts[:5000], s[:5000]), chunks
        pts2 = orc.g2_chain(4500, k, d)
        ctx.set_msm_chunks(4)
        assert ctx.g2_msm_device(to_dev(pts2), to_dev(s[:4500]), 4500) == orc.g2_msm(pts2, s[:4500])
    finally:
        ctx.set_msm_chunks(0)
        ctx.bases_free(h)
        ctx.bases_free(ht)


def test_ntt_2_26_roundtrip_and_direct_evaluation(ctx):
    """beyond the oracle's reach in full: round trip + a few outputs against the O(n) definition (config #3 property check)."""
    import torch
    log_n, n = 26, 1 << 26
    d = dev_empty(4 * n)
    ctx.fr_random_device(d, n, pyref.SEED_NTT, 12345, eb.SCALARS_MONT)
    orig = d.clone()
    ctx.fr_ntt_device(d, log_n, 0)
    host_in = to_host(orig).reshape(n, 4)
    out = to_host(d).reshape(n, 4)
    for kk in (0, 1, (1 << 25) + 12345, n - 1):
        assert (orc.fr_ntt_eval_output(host_in, log_n, kk) == out[kk]).all(), kk
    ctx.fr_ntt_device(d, log_n, eb.NTT_INVERSE)
    assert torch.equal(d, orig)


def test_gpu_msm_on_reference_kat_points_is_bilinear(ctx):
    """GPU MSMs over the points of the reference's own pairing KATs (tests/golden/pairing_kats.json, BE entry
    point): the results satisfy e(sum s_i P_i, Q) = prod e(P_i, s_i Q) under the pairing that replays those KATs."""
    import json, os
    kats = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "pairing_kats.json")))
    g1s, g2s = [], []
    for v in kats["vectors"][:6]:
        data = bytes.fromhex(v["calldata"])
        for i in range(0, len(data), 192):
            g1, g2 = pyref.g1_from_be(data[i:i + 64]), pyref.g2_from_be(data[i + 64:i + 192])
            if g1 is not None:
                g1s.append(g1)
            if g2 is not None:
                g2s.append(g2)
    g1s, g2s = g1s[:8], g2s[:4]
    s = [pyref.rand_fr(91, i) for i in range(8)]
    sbe = b"".join(pyref.fr_to_be(x) for x in s)
    a = ctx.g1_msm(b"".join(pyref.g1_to_be(p) for p in g1s), sbe, len(g1s), eb.POINTS_BE | eb.SCALARS_BE)
    assert a == orc.g1_msm(orc.g1_be_to_native(b"".join(pyref.g1_to_be(p) for p in g1s)), orc.ints_to_array(s))
    q = pyref.G2_GEN
    assert pyref.pairing_check([(pyref.g1_from_be(a), q)] + [(pyref.pt_neg(pyref._Fq, p), pyref.g2_mul(x, q)) for p, x in zip(g1s, s)])
    b = ctx.g2_msm(b"".join(pyref.g2_to_be(p) for p in g2s), sbe[:32 * len(g2s)], len(g2s), eb.POINTS_BE | eb.SCALARS_BE)
    pneg = pyref.pt_neg(pyref._Fq, pyref.G1_GEN)
    assert pyref.pairing_check([(pyref.G1_GEN, pyref.g2_from_be(b))] + [(pyref.g1_mul(x, pneg), p) for x, p in zip(s, g2s)])


def test_misaligned_device_buffers_are_rejected(ctx):
    """16-byte alignment is a precondition of the 128-bit loads / bulk copies: violating it is an error, not UB."""
    import torch
    buf = torch.zeros(4 * 64 + 1, dtype=torch.int64, device="cuda")
    pts = torch.zeros(8 * 64, dtype=torch.int64, device="cuda")
    with pytest.raises(eb.B200Error) as e:
        ctx.g1_msm_device(pts, buf[1:], 64)     # 8-byte aligned scalars
    assert e.value.status == 4
    with pytest.raises(eb.B200Error) as e:
        ctx.fr_ntt_device(buf[1:1 + 4 * 64], 6, 0)
    assert e.value.status == 4


# ---- batched precompile arithmetic: the reference's own vectors through the C ABI ---------------------------------
def _kats():
    import json
    return json.load(open(os.path.join(os.path.dirname(__file__), "golden", "pairing_kats.json")))


@pytest.mark.gpu
def test_pairing_check_matches_all_reference_kats(ctx):
    """The 14 ecpairing vectors of /root/reference/test/tests/levm/precompile_tests.rs:17-140, one batch, through
    b200zk_bn254_pairing_check_batch: expected booleans are the reference's, not the oracle's."""
    kats = _kats()
    checks = [bytes.fromhex(v["calldata"]) for v in kats["vectors"]]
    res, st = ctx.bn254_pairing_check_batch(checks)
    assert st == [0] * len(checks)
    assert res == [v["expected"] for v in kats["vectors"]], [v["name"] for v, r in zip(kats["vectors"], res) if r != v["expected"]]


@pytest.mark.gpu
def test_pairing_check_error_cases(ctx):
    kats = _kats()
    good = bytes.fromhex(kats["vectors"][0]["calldata"])
    oob = bytes.fromhex(kats["coordinate_out_of_bounds_calldata"])  # precompile_tests.rs:143-151
    oob = oob[:192 * (len(oob) // 192)]
    # a G1 point off the curve, a G2 point off the curve, and a G2 point on the twist but outside the r-subgroup
    bad_g1 = (1).to_bytes(32, "big") + (3).to_bytes(32, "big") + good[64:192]
    bad_g2 = good[:64] + good[64:160] + (int.from_bytes(good[160:192], "big") ^ 1).to_bytes(32, "big")
    outside = good[:64] + pyref.g2_to_be(_twist_point_outside_subgroup())  # on the twist, not in the r-subgroup
    res, st = ctx.bn254_pairing_check_batch([good, oob, bad_g1, bad_g2, outside, b"", good + bad_g1, oob + bad_g1])
    assert st == [0, 2, 3, 3, 3, 0, 3, 2]
    assert res == [1, 0, 0, 0, 0, 1, 0, 0]
    # identities on either side contribute one
    zero_g1 = bytes(64) + good[64:192]
    zero_g2 = good[:64] + bytes(128)
    res, st = ctx.bn254_pairing_check_batch([zero_g1, zero_g2, zero_g1 + good])
    assert st == [0, 0, 0] and res == [1, 1, 1]


def _fq_sqrt(v):
    r = pow(v, (pyref.P + 1) // 4, pyref.P)
    return r if r * r % pyref.P == v % pyref.P else None


def _f2_sqrt(a):
    """square root in Fq2 = Fq[u]/(u^2+1) by the norm method, or None"""
    P = pyref.P
    if a[1] == 0:
        r = _fq_sqrt(a[0])
        if r is not None:
            return (r, 0)
        r = _fq_sqrt(-a[0] % P)
        return None if r is None else (0, r)
    s = _fq_sqrt((a[0] * a[0] + a[1] * a[1]) % P)
    if s is None:
        return None
    half = pow(2, -1, P)
    for t in ((a[0] + s) * half % P, (a[0] - s) * half % P):
        x0 = _fq_sqrt(t)
        if x0:
            r = (x0, a[1] * pow(2 * x0, -1, P) % P)
            if pyref.f2_mul(r, r) == (a[0] % P, a[1] % P):
                return r
    return None


def _twist_point_outside_subgroup():
    for x in range(1, 400):  # bounded: about half of the x values give a twist point, nearly all of them outside
        rhs = pyref.f2_add(pyref.f2_mul(pyref.f2_mul((x, 1), (x, 1)), (x, 1)), pyref.B_G2)
        y = _f2_sqrt(rhs)
        pt = ((x, 1), y)
        # pyref.g2_mul reduces its scalar mod r, so r*pt is spelled (r-1)*pt + pt
        if y is not None and pyref.g2_on_curve(pt) and pyref.g2_add(pyref.g2_mul(pyref.R - 1, pt), pt) is not None:
            return pt
    raise AssertionError("no twist point found")


@pytest.mark.gpu
def test_pairing_check_bilinearity_on_fresh_points(ctx):
    """e(aP, bQ) * e(-(ab)P, Q) == 1 for scalars the KATs never saw; a perturbed product is not one."""
    import random
    rng = random.Random(0xB200)
    checks, want = [], []
    for k in range(6):
        a, b = rng.randrange(1, pyref.R), rng.randrange(1, pyref.R)
        lhs = pyref.g1_to_be(pyref.g1_mul(a, pyref.G1_GEN)) + pyref.g2_to_be(pyref.g2_mul(b, pyref.G2_GEN))
        good = pyref.g1_to_be(pyref.g1_mul(pyref.R - (a * b) % pyref.R, pyref.G1_GEN)) + pyref.g2_to_be(pyref.G2_GEN)
        bad = pyref.g1_to_be(pyref.g1_mul(pyref.R - (a * b + 1 + k) % pyref.R, pyref.G1_GEN)) + pyref.g2_to_be(pyref.G2_GEN)
        checks += [lhs + good, lhs + bad]
        want += [1, 0]
    res, st = ctx.bn254_pairing_check_batch(checks)
    assert st == [0] * len(checks) and res == want


@pytest.mark.gpu
def test_g1_add_mul_batch_vs_reference_kats_and_oracle(ctx):
    g = pyref.g1_to_be(pyref.G1_GEN)
    seven_g = bytes.fromhex("17072b2ed3bb8d759a5325f477629386cb6fc6ecb801bd76983a6b86abffe078"
                            "168ada6cd130dd52017bb54bfa19377aadfe3bf05d18f41b77809f7f60d4af9e")  # integration_tests.rs:572
    two_g = bytes.fromhex("030644e72e131a029b85045b68181585d97816a916871ca8d3c208c16d87cfd3"
                          "15ed738c0e0a7c92e7845f96b2ae9c0a68a6a449e3538fc7ff3ebf7a5a18a2c4")
    neg_g = pyref.g1_to_be((1, pyref.P - 2))
    off = (1).to_bytes(32, "big") + (3).to_bytes(32, "big")
    big = pyref.P.to_bytes(32, "big") + (2).to_bytes(32, "big")
    # ecMul: 7*G (the reference's own KAT), r*G = identity, 0*G, k*identity, (2^256-1)*G, off-curve, out of range
    pts = g + g + g + bytes(64) + g + off + big
    ks = [7, pyref.R, 0, 5, (1 << 256) - 1, 3, 3]
    out, st = ctx.bn254_g1_mul_batch(pts, b"".join(k.to_bytes(32, "big") for k in ks))
    assert st == [0, 1, 1, 1, 0, 3, 2]
    assert out[:64] == seven_g and out[64:256] == bytes(192)
    assert out[256:320] == pyref.g1_to_be(pyref.g1_mul(((1 << 256) - 1) % pyref.R, pyref.G1_GEN))
    assert out[320:] == bytes(128)
    # ecAdd: G+G (doubling), G+(-G) (cancellation), G+0, 0+0, 2G+7G vs the oracle, off-curve, out of range
    a = g + g + g + bytes(64) + two_g + off + g
    b = g + neg_g + bytes(64) + bytes(64) + seven_g + g + big
    out, st = ctx.bn254_g1_add_batch(a, b)
    assert st == [0, 1, 0, 1, 0, 3, 2]
    assert out[:64] == two_g and out[64:128] == bytes(64) and out[128:192] == g and out[192:256] == bytes(64)
    rc, nine_g = orc.g1_add_be(two_g, seven_g)
    assert out[256:320] == nine_g == pyref.g1_to_be(pyref.g1_mul(9, pyref.G1_GEN))
    # a larger random batch against the C++ oracle
    n = 300
    s = orc.rand_fr(0xB2000009, 0, 2 * n)
    pa = [orc.g1_mul_be(g, orc.limbs_to_int(s[i]).to_bytes(32, "big"))[1] for i in range(n)]
    kb = [orc.limbs_to_int(s[n + i]).to_bytes(32, "big") for i in range(n)]
    out, st = ctx.bn254_g1_mul_batch(b"".join(pa), b"".join(kb))
    assert st == [0] * n
    for i in range(0, n, 17):
        assert out[64 * i:64 * i + 64] == orc.g1_mul_be(pa[i], kb[i])[1]
    out, st = ctx.bn254_g1_add_batch(b"".join(pa), b"".join(reversed(pa)))
    assert st == [0] * n
    for i in range(0, n, 13):
        assert out[64 * i:64 * i + 64] == orc.g1_add_be(pa[i], pa[n - 1 - i])[1]


@pytest.mark.gpu
@pytest.mark.parametrize("log_n", [3, 6])
def test_real_groth16_proof_from_the_gpu_pipeline_verifies(ctx, log_n):
    """A real Groth16 instance (tests/groth16_toy.py: random R1CS, trusted setup with known toxic waste): the GPU
    pipeline (3 iNTT + 3 coset NTT + quotient + coset iNTT, 4 G1 MSMs + 1 G2 MSM over the caller's proving key)
    must produce the proof BIT FOR BIT as computed in the exponent, and the Groth16 verification equation must hold
    under the GPU pairing check (itself pinned by the reference's ecpairing vectors)."""
    from ethrex_b200.groth16 import Groth16Prover
    from groth16_toy import N_PUBLIC, ToyGroth16
    toy = ToyGroth16(log_n)
    prover = Groth16Prover(ctx, log_n, toy.a_g1, toy.b_g1, toy.b_g2, toy.l_g1, toy.h_g1, N_PUBLIC)
    try:
        checks, want = [], []
        for x in (7, pyref.R - 5):
            z = toy.assign(x)
            a, b, c = toy.evaluations(z)
            proof = prover.prove(z, a, b, c)
            assert proof == toy.expected_proof(z)
            tampered = proof[:192] + pyref.g1_to_be(pyref.g1_add(pyref.g1_from_be(proof[192:256]), pyref.G1_GEN))
            checks += [toy.verifier_calldata(proof, x), toy.verifier_calldata(proof, x + 1), toy.verifier_calldata(tampered, x)]
            want += [1, 0, 0]
        res, st = ctx.bn254_pairing_check_batch(checks)
        assert st == [0] * len(checks) and res == want
    finally:
        prover.close()


@pytest.mark.gpu
def test_c_abi_from_plain_c():
    """examples/c_abi_demo.c: the boundary used from C with nothing but include/b200zk.h and libb200zk.so in the
    process (what a cgo / Rust FFI binding does) -- reference KATs, error statuses, NTT round trip."""
    import subprocess
    exe = os.path.join(os.path.dirname(os.path.dirname(__file__)), "examples", "build", "c_abi_demo")
    assert os.path.exists(exe), "build it with `python -c 'import __graft_entry__ as g; g.build()'`"
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "all checks passed" in r.stdout


@pytest.mark.gpu
def test_groth16_commit_from_plain_c(tmp_path):
    """b200zk_groth16_commit driven from C only (examples/c_abi_demo.c section 6): a real Groth16 instance (trusted
    setup with known toxic waste, tests/groth16_toy.py) uploaded once, proved in ONE call, bit-exact against the proof
    computed in the exponent -- the orchestration a Rust / cgo caller gets without re-implementing it."""
    import subprocess
    from groth16_toy import write_c_fixture
    exe = os.path.join(os.path.dirname(os.path.dirname(__file__)), "examples", "build", "c_abi_demo")
    assert os.path.exists(exe), "build it with `python -c 'import __graft_entry__ as g; g.build()'`"
    fx = str(tmp_path / "groth16_toy_2_4.bin")
    write_c_fixture(fx, log_n=4)
    r = subprocess.run([exe, fx], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "b200zk_groth16_commit == the proof computed in the exponent" in r.stdout and "all checks passed" in r.stdout


@pytest.mark.gpu
@pytest.mark.parametrize("precompute", [False, True])
def test_multi_msm_shares_one_sort_and_matches_single_calls(ctx, precompute):
    """b200zk_msm_multi_resident_device (Groth16's witness MSMs): G1, G1, G2, G1 columns against one scalar vector
    give exactly the results of four separate resident MSMs, which are checked against the closed form."""
    import torch
    n = 1 << 14
    cols = []
    for tag, g2 in ((3, False), (5, False), (7, True), (11, False)):
        k, d = (chain_kd()[0] * tag) % pyref.R, (chain_kd()[1] + tag) % pyref.R
        pts = torch.empty((16 if g2 else 8) * n, dtype=torch.int64, device="cuda")
        (ctx.g2_chain_device if g2 else ctx.g1_chain_device)(pts, 0, n, k, d)
        h = (ctx.g2_bases_from_device if g2 else ctx.g1_bases_from_device)(pts, n)
        if precompute:
            ctx.bases_precompute(h, 0)
        cols.append((h, g2, k, d))
    try:
        for m in (n, n - 37, 2, 1):
            s = scalars_special(m)
            ds = to_dev(s)
            multi = ctx.msm_multi_resident_device([c[0] for c in cols], [c[1] for c in cols], ds, m)
            for (h, g2, k, d), got in zip(cols, multi):
                single = (ctx.g2_msm_resident_device if g2 else ctx.g1_msm_resident_device)(h, ds, m)
                assert got == single
                assert got == (expected_chain_msm_g2 if g2 else expected_chain_msm_g1)(s, k, d)
        # a zero vector: every column's result is the identity
        z = to_dev(np.zeros((8, 4), dtype=np.uint64))
        multi = ctx.msm_multi_resident_device([c[0] for c in cols], [c[1] for c in cols], z, 8)
        assert multi == [bytes(128 if c[1] else 64) for c in cols]
        # mixing a precomputed and a plain column is refused
        if precompute:
            pts = torch.empty(8 * n, dtype=torch.int64, device="cuda")
            ctx.g1_chain_device(pts, 0, n, 3, 5)
            plain = ctx.g1_bases_from_device(pts, n)
            with pytest.raises(eb.B200Error) as e:
                ctx.msm_multi_resident_device([cols[0][0], plain], [False, False], to_dev(scalars_special(8)), 8)
            assert e.value.status == 4
            ctx.bases_free(plain)
    finally:
        for c in cols:
            ctx.bases_free(c[0])


@pytest.mark.gpu
def test_msm_entry_points_report_the_identity_as_status_1(ctx):
    """ZisK-style status table (crates/guest-program/src/crypto/zisk.rs:144-172): 1 = ok, result is the point at
    infinity.  Checked on the raw return codes of the host, device and resident entry points, G1 and G2."""
    import ctypes as C
    from ethrex_b200 import _ffi as F
    g, g2 = pyref.g1_to_be(pyref.G1_GEN), pyref.g2_to_be(pyref.G2_GEN)
    five, rm5, one = (5).to_bytes(32, "big"), (pyref.R - 5).to_bytes(32, "big"), (1).to_bytes(32, "big")
    flags = eb.POINTS_BE | eb.SCALARS_BE
    out = C.create_string_buffer(128)
    for pts, fn, size in ((g + g, F.lib.b200zk_g1_msm, 64), (g2 + g2, F.lib.b200zk_g2_msm, 128)):
        assert fn(ctx._h, pts, five + rm5, 2, flags, out) == 1 and out.raw[:size] == bytes(size)
        assert fn(ctx._h, pts, five + one, 2, flags, out) == 0 and out.raw[:size] != bytes(size)
        assert fn(ctx._h, pts, five + rm5, 0, flags, out) == 1 and out.raw[:size] == bytes(size)  # empty sum
    h = ctx.g1_bases_upload(g + g, 2, eb.POINTS_BE)
    assert F.lib.b200zk_g1_msm_resident(ctx._h, h, five + rm5, 2, eb.SCALARS_BE, out) == 1
    assert F.lib.b200zk_g1_msm_resident(ctx._h, h, five + one, 2, eb.SCALARS_BE, out) == 0
    ctx.bases_free(h)


@pytest.mark.gpu
def test_groth16_golden_fixture(ctx):
    """tests/golden/groth16_toy.json (made by make_groth16_golden.py on the CPU oracle): the GPU prover reproduces
    the committed proof bytes, and the committed verifier calldata passes the GPU pairing check."""
    import json
    from ethrex_b200.groth16 import Groth16Prover
    from groth16_toy import N_PUBLIC, ToyGroth16
    gold = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "groth16_toy.json")))
    for inst in gold["instances"]:
        toy = ToyGroth16(inst["log_n"])
        prover = Groth16Prover(ctx, inst["log_n"], toy.a_g1, toy.b_g1, toy.b_g2, toy.l_g1, toy.h_g1, N_PUBLIC)
        try:
            for case in inst["cases"]:
                x = int(case["public_input"], 16)
                z = toy.assign(x)
                assert prover.prove(z, *toy.evaluations(z)).hex() == case["proof"]
            res, st = ctx.bn254_pairing_check_batch([bytes.fromhex(c["verifier_calldata"]) for c in inst["cases"]])
            assert st == [0] * len(res) and res == [1] * len(res)
        finally:
            prover.close()


@pytest.mark.gpu
def test_groth16_verifier_batch_on_the_gpu(ctx):
    """Groth16Verifier (what ProverBackend::verify / the on-chain verifier compute): proofs from the GPU prover for
    several public inputs verify in one batch; a wrong public input, a tampered proof and a proof with a point off
    the curve do not.  B200Backend.verify maps the outcome to Ok / BackendError::Verification."""
    from ethrex_b200.backend import B200Backend, B200ProveOutput, ProverType
    from ethrex_b200.groth16 import Groth16Prover, Groth16Verifier
    from groth16_toy import N_PUBLIC, ToyGroth16, _g1
    toy = ToyGroth16(4)
    prover = Groth16Prover(ctx, 4, toy.a_g1, toy.b_g1, toy.b_g2, toy.l_g1, toy.h_g1, N_PUBLIC)
    ver = Groth16Verifier(ctx, toy.vk_alpha_g1, toy.vk_beta_g2, toy.vk_gamma_g2, toy.vk_delta_g2, [_g1(s) for s in toy.ic])
    try:
        xs = [3, 0, pyref.R - 1, 0xDEADBEEF]
        proofs = []
        for x in xs:
            z = toy.assign(x)
            proofs.append(prover.prove(z, *toy.evaluations(z)))
        assert ver.verify_batch(proofs, [[x] for x in xs]) == [True] * 4
        assert ver.verify_batch(proofs, [[x + 1] for x in xs]) == [False] * 4
        assert ver.verify_batch([proofs[1], proofs[0]], [[xs[0]], [xs[1]]]) == [False, False]
        off_curve = proofs[0][:63] + bytes([proofs[0][63] ^ 1]) + proofs[0][64:]
        assert ver.verify(off_curve, [xs[0]]) is False
        backend = B200Backend(ctx, verifier=ver)
        out = B200ProveOutput(ProverType.SP1, proofs[2], {})
        backend.verify(out, [xs[2]])
        with pytest.raises(eb.B200Error) as e:
            backend.verify(out, [xs[3]])
        assert e.value.kind == "Verification"
        with pytest.raises(eb.B200Error):
            B200Backend(ctx).verify(out, [xs[2]])  # no verifier: "Verify not implemented for this backend"
    finally:
        prover.close()
