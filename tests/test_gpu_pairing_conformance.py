"""Both pairings stage by stage on the device, and every subgroup check against points of each cofactor order.

tests/csrc/pairing_conformance.cu runs one stage per thread (built into the conformance library by
ethrex_b200/csrc/Makefile with the library's own nvcc flags); tests/pairing_stages_ref.py restates each stage in Python,
and tests/test_pairing_stages_host.py ties that restatement to independent anchors (f^p, f^x, the generic final power,
[|x|]Q, the independent pairing of bls_pairing_ref, bilinearity).  Every stage compares bit for bit.

The second half feeds points whose order is one prime l of the cofactor (and the largest l-power order the group holds,
and those plus a subgroup point) to the harness's subgroup checks and to every entry point that checks the subgroup:
each must return its documented status 3 with its valid neighbours intact.  EIP-2537 addition has no subgroup check,
so it must add these points like any other."""
import ctypes
import os
import random

import numpy as np
import pytest

import bls_pairing_ref as B
import bls_ref as bls
import field_conformance_ref as ref
import pairing_stages_ref as S
import pyref
import pyref_tower as BT

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "build", "libb200zk_conformance.so")
T_BLS, T_BN = 0, 1
OPS = ["frob", "frob2", "exp_x", "final_exp", "line_double", "line_add", "g2_prepare", "miller", "pair", "in_subgroup_g1",
       "in_subgroup_g2", "line_at", "miller_ate"]
OP = {name: i for i, name in enumerate(OPS)}
N_XCHAIN = 1 << 10  # the x-chain final exponentiation restated in Python: about 45 ms per item
FP, FP2, F12 = ref.FP381, ref.FP2_381, ref.BLS_FP12
FQ, FQ2, Q12 = ref.FQ, ref.FQ2, ref.BN_FP12


@pytest.fixture(scope="module")
def run():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    assert os.path.exists(LIB), f"{LIB} is missing: run __graft_entry__.build() first"
    torch.cuda.set_device(0)
    fn = ctypes.CDLL(LIB).b200zk_pairing_conformance_run
    fn.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint64]
    fn.restype = ctypes.c_int

    def go(tid, op, cols, out_words):
        arr = np.ascontiguousarray(np.concatenate(cols, axis=1), dtype=np.uint32)
        n, iw = arr.shape
        d_in = torch.from_numpy(arr.view(np.int32)).cuda()
        d_out = torch.zeros((n, out_words), dtype=torch.int32, device="cuda")
        rc = fn(tid, OP[op] if isinstance(op, str) else op, d_in.data_ptr(), iw, d_out.data_ptr(), out_words, n)
        assert rc == 0, f"b200zk_pairing_conformance_run(type {tid}, op {op}) returned {rc}"
        return d_out.cpu().numpy().view(np.uint32)
    return go


# ---- encodings: semantic values -> raw Montgomery limbs and back ---------------------------------------------------------
def enc12(T, vals):
    return ref.pack_elems(T, [T.enc(v) for v in vals])


def dec12(T, arr):
    return [T.dec(x) for x in ref.unpack_elems(T, arr)]


def enc_f2(F2, vals):
    return ref.pack_elems(F2, [F2.enc(v) for v in vals])


def dec_f2(F2, arr):
    return [F2.dec(x) for x in ref.unpack_elems(F2, arr)]


def enc_g1(F, pts):  # affine (x, y), the identity (0, 0)
    return np.concatenate([ref.pack_elems(F, [F.enc(0 if p is None else p[k]) for p in pts]) for k in range(2)], axis=1)


def enc_g2(F2, pts):
    return np.concatenate([enc_f2(F2, [(0, 0) if q is None else q[k] for q in pts]) for k in range(2)], axis=1)


def dec_lines(arr, n_lines):
    """(n, 72 n_lines) words -> per item, n_lines triples of Fp2"""
    f2 = dec_f2(FP2, arr.reshape(-1, FP2.words))
    per = 3 * n_lines
    return [[tuple(f2[i * per + 3 * k:i * per + 3 * k + 3]) for k in range(n_lines)] for i in range(len(arr))]


def assert_equal(what, inputs, got, exp):
    bad = [i for i, (g, e) in enumerate(zip(got, exp)) if g != e]
    assert not bad, f"{what}: {len(bad)} of {len(exp)} differ, first at item {bad[0]}: input {inputs[bad[0]]!r}"


# ---- inputs -------------------------------------------------------------------------------------------------------------
def _f12(cs):
    """six Fp2 coefficients of w^0 .. w^5 -> tower"""
    return S._tower(cs)


def edge_f12():
    """the field-conformance edges lifted to Fp12: zero, one, all coefficients p - 1, one nonzero coordinate at each of the
    12 slots (1, p - 1, R mod p), -1, w, and elements of the subfields Fp, Fp2, Fp6"""
    p, Rm = S.P, (1 << 384) % S.P
    z = (0, 0)
    out = [S.ZERO, S.ONE, _f12([(p - 1, p - 1)] * 6), _f12([(p - 1, 0)] + [z] * 5), S.W]
    for k in range(6):
        for c in (0, 1):
            for v in (1, p - 1, Rm):
                cs = [z] * 6
                cs[k] = (v, 0) if c == 0 else (0, v)
                out.append(_f12(cs))
    out += [_f12([(v, 0)] + [z] * 5) for v in (2, (p - 1) // 2, Rm)]  # Fp
    out += [_f12([(3, 5)] + [z] * 5), _f12([(p - 1, 1)] + [z] * 5)]  # Fp2
    out.append((((7, 1), (2, p - 3), (11, 13)), (z, z, z)))  # Fp6: no odd powers of w
    return out


def random_f12(rng, n):
    return [_f12([(rng.randrange(S.P), rng.randrange(S.P)) for _ in range(6)]) for _ in range(n)]


def subfield_one(f):
    """f lies in Fp6 (hence in Fp, Fp2): the final exponentiation gives exactly 1"""
    return f != S.ZERO and f[1] == ((0, 0),) * 3


# ---- BLS12-381 stages ----------------------------------------------------------------------------------------------------
def test_bls_frobenius(run):
    rng = random.Random("frob")
    items = edge_f12() + random_f12(rng, N_XCHAIN)
    for op, fn in (("frob", S.frob), ("frob2", S.frob2)):
        got = dec12(F12, run(T_BLS, op, [enc12(F12, items)], F12.words))
        assert_equal(f"bls {op}", items, got, [fn(a) for a in items])


def test_bls_exp_x(run):
    """cyclotomic inputs (where the result is f^x) and arbitrary ones (where it is conj(f^|x|))"""
    rng = random.Random("exp_x")
    easy = lambda f: S.mul(S.frob2(S.mul(S.conj(f), S.inv(f))), S.mul(S.conj(f), S.inv(f)))  # noqa: E731
    cyc = [S.ONE] + [easy(f) for f in random_f12(rng, N_XCHAIN // 2)]
    items = cyc + edge_f12() + random_f12(rng, N_XCHAIN // 2)
    got = dec12(F12, run(T_BLS, "exp_x", [enc12(F12, items)], F12.words))
    assert_equal("bls exp_x", items, got, [S.exp_x(a) for a in items])
    for c, r in zip(cyc[:8], got[:8]):
        assert S.mul(r, S.power(c, S.X_ABS)) == S.ONE  # f^x f^|x| = 1


def test_bls_final_exponentiation(run):
    rng = random.Random("final_exp")
    lines = S.g2_prepare(B.g2_mul(5, B.G2))[0]
    millers = [S.miller(lines, bls.mul(k, B.G1)) for k in (1, 2, S.R - 1)]
    items = edge_f12() + millers + random_f12(rng, N_XCHAIN)
    got = dec12(F12, run(T_BLS, "final_exp", [enc12(F12, items)], F12.words))
    exp = [S.final_exponentiate(a) for a in items]
    assert_equal("bls final_exponentiate", items, got, exp)
    assert got[0] == S.ZERO  # f = 0 gives 0: inv(0) = 0 carries through
    for f, r in zip(items, got):
        if subfield_one(f):
            assert r == S.ONE, f
    # the independent anchor on a few device outputs: the generic power 3 (p^12 - 1)/r
    for f, r in list(zip(items, got))[3:5] + list(zip(millers, got[len(edge_f12()):]))[:1]:
        assert r == S.power(f, S.FINAL_EXP_BLS)


def _random_proj(rng, q):
    """q in homogeneous coordinates with a random Z"""
    z = (rng.randrange(1, S.P), rng.randrange(S.P))
    return (B.f2_mul(q[0], z), B.f2_mul(q[1], z), z)


def _g2_points(rng):
    g = B.G2
    return [g, B.g2_neg(g), B.g2_mul(S.R - 1, g), B.g2_mul(2, g), B.g2_mul(3, g)] + [B.g2_mul(rng.randrange(1, S.R), g) for _ in range(3)]


def _enc_proj(Ts):
    return np.concatenate([enc_f2(FP2, [T[k] for T in Ts]) for k in range(3)], axis=1)


def _dec_proj_line(out):
    f2 = [dec_f2(FP2, out[:, k * FP2.words:(k + 1) * FP2.words]) for k in range(6)]
    return [(tuple(c[i] for c in f2[:3]), tuple(c[i] for c in f2[3:])) for i in range(len(out))]


def test_bls_line_double_and_add(run):
    rng = random.Random("lines")
    qs = _g2_points(rng)
    Ts = [(q[0], q[1], (1, 0)) for q in qs] + [_random_proj(rng, q) for q in qs for _ in range(4)]
    Ts += [_random_proj(rng, B.g2_random_point(s)) for s in range(8)]  # on the twist, outside G2: the formulas do not care
    out = run(T_BLS, "line_double", [_enc_proj(Ts)], 6 * FP2.words)
    assert_equal("bls line_double", Ts, _dec_proj_line(out), [S.line_double(T) for T in Ts])
    adds = [(T, rng.choice(qs)) for T in Ts]
    out = run(T_BLS, "line_add", [_enc_proj([T for T, _ in adds]), enc_g2(FP2, [q for _, q in adds])], 6 * FP2.words)
    assert_equal("bls line_add", adds, _dec_proj_line(out), [S.line_add(T, q) for T, q in adds])


def test_bls_prepare_miller_pair(run):
    rng = random.Random("miller")
    qs = _g2_points(rng)
    prepared = [S.g2_prepare(q)[0] for q in qs]
    got = dec_lines(run(T_BLS, "g2_prepare", [enc_g2(FP2, qs)], 68 * 3 * FP2.words), 68)
    assert_equal("bls g2_prepare", qs, got, prepared)
    g = B.G1
    ps = [g, (g[0], S.P - g[1]), bls.mul(S.R - 1, g), bls.mul(2, g), bls.mul(3, g)] + [bls.mul(rng.randrange(1, S.R), g) for _ in range(3)]
    items = [(k, p) for k in range(len(qs)) for p in ps]
    line_cols = np.stack([ref.pack_elems(FP2, [FP2.enc(c) for l in prepared[k] for c in l]).reshape(-1) for k, _ in items])
    got = dec12(F12, run(T_BLS, "miller", [line_cols, enc_g1(FP, [p for _, p in items])], F12.words))
    assert_equal("bls miller", items, got, [S.miller(prepared[k], p) for k, p in items])
    pairs = [(p, qs[k]) for k, p in items[::3]]
    out = run(T_BLS, "pair", [enc_g1(FP, [p for p, _ in pairs]), enc_g2(FP2, [q for _, q in pairs])], F12.words + 68 * 3 * FP2.words)
    got = dec12(F12, out[:, :F12.words])
    assert_equal("bls pair", pairs, got, [S.pair(p, q) for p, q in pairs])
    assert dec_lines(out[:, F12.words:], 68) == [S.g2_prepare(q)[0] for _, q in pairs]


def test_bls_pair_anchors(run):
    """bilinearity on the device, e(aP, bQ) = e(P, Q)^(ab), and the device pairing is the inverse cube of the independent
    pairing of bls_pairing_ref (its x-chain yields the cube, and x < 0 conjugates the Miller value)"""
    rng = random.Random("bilinear")
    ab = [(rng.randrange(1, S.R), rng.randrange(1, S.R)) for _ in range(4)] + [(S.R - 1, 1), (2, S.R - 1)]
    pairs = [(B.G1, B.G2)] + [(bls.mul(a, B.G1), B.g2_mul(b, B.G2)) for a, b in ab]
    out = run(T_BLS, "pair", [enc_g1(FP, [p for p, _ in pairs]), enc_g2(FP2, [q for _, q in pairs])], F12.words + 68 * 3 * FP2.words)
    got = dec12(F12, out[:, :F12.words])
    e = got[0]
    assert e != S.ONE and S.power(e, S.R) == S.ONE
    for (a, b), r in zip(ab, got[1:]):
        assert r == S.power(e, a * b % S.R)
    assert e == S.inv(S.power(S.from_flat(B.pairing(B.G1, B.G2)), 3))


# ---- BN254 stages ---------------------------------------------------------------------------------------------------------
def _bn_points(rng):
    g1, g2 = pyref.G1_GEN, pyref.G2_GEN
    ps = [g1, pyref.g1_mul(pyref.R - 1, g1), pyref.g1_mul(2, g1)] + [pyref.g1_mul(rng.randrange(1, pyref.R), g1) for _ in range(3)]
    qs = [g2, pyref.g2_mul(pyref.R - 1, g2), pyref.g2_mul(3, g2)] + [pyref.g2_mul(rng.randrange(1, pyref.R), g2) for _ in range(3)]
    return ps, qs


def test_bn_line_at(run):
    rng = random.Random("line_at")
    p_ = pyref.P
    r2 = lambda: (rng.randrange(p_), rng.randrange(p_))  # noqa: E731
    ps, _ = _bn_points(rng)
    items = [(r2(), r2(), r2(), rng.choice(ps)) for _ in range(1024)] + [((0, 0), (0, 0), (0, 0), ps[0]), ((p_ - 1, p_ - 1), (1, 0), (0, 1), ps[1])]
    cols = [enc_f2(FQ2, [it[k] for it in items]) for k in range(3)] + [enc_g1(FQ, [it[3] for it in items])]
    got = dec12(Q12, run(T_BN, "line_at", cols, Q12.words))
    assert_equal("bn line_at", items, got, [BT._line(lam, xt, yt, p) for lam, xt, yt, p in items])


def test_bn_miller_final_pair(run):
    rng = random.Random("bn_pair")
    ps, qs = _bn_points(rng)
    items = [(p, q) for p in ps for q in qs[:4]]
    cols = [enc_g1(FQ, [p for p, _ in items]), enc_g2(FQ2, [q for _, q in items])]
    millers = dec12(Q12, run(T_BN, "miller_ate", cols, Q12.words))
    assert_equal("bn miller_ate", items, millers, [BT.miller_ate(q, p) for p, q in items])
    pairs = dec12(Q12, run(T_BN, "pair", [enc_g1(FQ, [p for p, _ in items[:8]]), enc_g2(FQ2, [q for _, q in items[:8]])], Q12.words))
    assert_equal("bn pair", items[:8], pairs, [BT.final_exponentiate(m) for m in millers[:8]])
    # bilinearity: e([a]P, [b]Q) = e(P, Q)^(ab)
    ab = [(rng.randrange(1, pyref.R), rng.randrange(1, pyref.R)) for _ in range(3)]
    bil = [(pyref.G1_GEN, pyref.G2_GEN)] + [(pyref.g1_mul(a, pyref.G1_GEN), pyref.g2_mul(b, pyref.G2_GEN)) for a, b in ab]
    got = dec12(Q12, run(T_BN, "pair", [enc_g1(FQ, [p for p, _ in bil]), enc_g2(FQ2, [q for _, q in bil])], Q12.words))
    assert got[0] != BT.F12_ONE
    for (a, b), r in zip(ab, got[1:]):
        assert r == BT.f12_pow(got[0], a * b % pyref.R)


def _bn_f12(rng, n):
    p_ = pyref.P
    return [tuple(tuple((rng.randrange(p_), rng.randrange(p_)) for _ in range(3)) for _ in range(2)) for _ in range(n)]


def test_bn_final_exponentiation(run):
    rng = random.Random("bn_final")
    p_, Rm = pyref.P, (1 << 256) % pyref.P
    z = (0, 0)
    edges = [BT.F12_ONE, (((p_ - 1, 0), z, z), (z, z, z)), (((p_ - 1, p_ - 1),) * 3, ((p_ - 1, p_ - 1),) * 3), ((z, z, z), ((1, 0), z, z))]
    for k in range(6):
        for c in (0, 1):
            cs = [z] * 6
            cs[k] = (Rm, 0) if c == 0 else (0, Rm)
            edges.append(((cs[0], cs[2], cs[4]), (cs[1], cs[3], cs[5])))
    edges += [(((3, 5), (7, 0), (0, 11)), (z, z, z))]  # Fp6
    items = edges + _bn_f12(rng, 48)
    zero = ((z, z, z), (z, z, z))
    got = dec12(Q12, run(T_BN, "final_exp", [enc12(Q12, items + [zero])], Q12.words))
    assert got[-1] == zero  # f = 0 gives 0
    assert_equal("bn final_exponentiate", items, got[:-1], [BT.final_exponentiate(f) for f in items])
    for f, r in zip(items, got):
        if f[1] == (z, z, z):
            assert r == BT.F12_ONE
    for f, r in list(zip(items, got))[-4:]:  # the independent anchor: the generic power (p^12 - 1)/r
        assert r == BT.f12_pow(f, (pyref.P ** 12 - 1) // pyref.R)


# ---- the subgroup checks against cofactor-component points -----------------------------------------------------------------
GROUPS = [(S.BLS_G1, T_BLS, "in_subgroup_g1", lambda pts: enc_g1(FP, pts)),
          (S.BLS_G2, T_BLS, "in_subgroup_g2", lambda pts: enc_g2(FP2, pts)),
          (S.BN_G2, T_BN, "in_subgroup_g2", lambda pts: enc_g2(FQ2, pts))]


@pytest.fixture(scope="module")
def cases():
    return {G.name: G.cases() for G, _, _, _ in GROUPS}


@pytest.mark.parametrize("G,tid,op,enc", GROUPS, ids=[G.name for G, _, _, _ in GROUPS])
def test_in_subgroup_every_component(run, cases, G, tid, op, enc):
    cs = cases[G.name]
    got = [int(v) for v in run(tid, op, [enc([pt for _, pt, _ in cs] + [None])], 1)[:, 0]]
    assert got[-1] == 1  # the identity
    wrong = [name for (name, _, want), g in zip(cs, got) if g != int(want)]
    assert not wrong, f"{G.name}: in_subgroup wrong for {wrong}"


def _off(cs):
    return [(name, pt) for name, pt, sub in cs if not sub]


def test_eip2537_pairing_rejects_every_component(ctx, cases):
    """bls_pair_decode, both sides: status 3 and result 0 next to valid checks"""
    valid = B.g1_eip2537(B.G1) + B.g2_eip2537(B.G2) + B.g1_eip2537(B.G1) + B.g2_eip2537(B.g2_neg(B.G2))
    bad = [B.g1_eip2537(pt) + B.g2_eip2537(B.G2) for _, pt in _off(cases["bls12_381_g1"])]
    bad += [B.g1_eip2537(B.G1) + B.g2_eip2537(pt) for _, pt in _off(cases["bls12_381_g2"])]
    checks = []
    for b in bad:
        checks += [valid, valid + b]
    checks.append(valid)
    res, st = ctx.bls12_381_pairing_check_batch(checks)
    assert st == [0, 3] * len(bad) + [0]
    assert res == [1, 0] * len(bad) + [1]


@pytest.mark.parametrize("gname", ["bls12_381_g1", "bls12_381_g2"])
def test_eip2537_msm_rejects_every_component(ctx, cases, gname):
    """bls_msm_terms: status 3 for the point under any scalar, zero included, and an all-zero output; valid neighbours intact"""
    import bls12_ops_ref as ops
    g = ops.G1 if gname == "bls12_381_g1" else ops.G2
    good = g.calldata([(g.mul(99, g.gen), 2), (g.gen, 3)])
    calls = []
    for _, pt in _off(cases[gname]):
        for k in (0, 1, S.R - 1):
            calls += [good, g.calldata([(g.gen, 5), (pt, k)])]
    calls.append(good)
    fn = ctx.bls12_381_g1_msm_batch if g is ops.G1 else ctx.bls12_381_g2_msm_batch
    outs, st = fn(calls)
    n = len(calls) // 2
    assert st == [0, 3] * n + [0]
    exp_good = g.encode(g.msm([(g.mul(99, g.gen), 2), (g.gen, 3)]))
    assert all(o == (exp_good if s == 0 else bytes(g.size)) for o, s in zip(outs, st))


@pytest.mark.parametrize("gname", ["bls12_381_g1", "bls12_381_g2"])
def test_eip2537_add_accepts_every_component(ctx, cases, gname):
    """EIP-2537 addition has no subgroup check: these points add like any other, to the oracle's sums"""
    import bls12_ops_ref as ops
    g = ops.G1 if gname == "bls12_381_g1" else ops.G2
    pts = [pt for _, pt, _ in cases[gname]]
    items = [(a, b) for a in pts for b in (pts[0], pts[-1], a, g.neg(a))]
    fn = ctx.bls12_381_g1_add_batch if g is ops.G1 else ctx.bls12_381_g2_add_batch
    out, st = fn(b"".join(g.encode(a) for a, _ in items), b"".join(g.encode(b) for _, b in items))
    for i, (a, b) in enumerate(items):
        s = g.add(a, b)
        assert (out[g.size * i:g.size * (i + 1)], st[i]) == (g.encode(s), 1 if s is None else 0), i


def test_g2_bases_upload_rejects_every_component(ctx, cases):
    """bls_g2_decode: status 3 for the compressed point alone and behind a valid one; the valid setup still uploads"""
    import ethrex_b200 as eb
    for name, pt in _off(cases["bls12_381_g2"]):
        for pts in (B.g2_compress(pt), B.G2_COMPRESSED + B.g2_compress(pt)):
            with pytest.raises(eb.B200Error) as e:
                ctx.bls12_381_g2_bases_upload(pts, len(pts) // 96)
            assert e.value.status == 3, name
    h = ctx.bls12_381_g2_bases_upload(B.G2_COMPRESSED + B.g2_compress(B.g2_mul(7, B.G2)), 2)
    ctx.bases_free(h)


def test_kzg_verify_rejects_every_component(ctx, cases):
    """bls_g1_decode_subgroup: a commitment or a proof of each component order gives status 3; valid items verify"""
    tau = 0x2F1B7C93D4A5E6F708192A3B4C5D6E7F8091A2B3C4D5E6F708192A3B4C5D6E7F % S.R
    g2 = ctx.bls12_381_g2_bases_upload(B.G2_COMPRESSED + B.g2_compress(B.g2_mul(tau, B.G2)), 2)
    try:
        poly = lambda x: (3 + 5 * x + 7 * x * x) % S.R  # noqa: E731
        z = 0x123456789
        y = poly(z)
        c = bls.compress(bls.mul(poly(tau), B.G1))
        pi = bls.compress(bls.mul((poly(tau) - y) * pow(tau - z, -1, S.R), B.G1))
        good = (c, z, y, pi)
        items, want = [], []
        for _, pt in _off(cases["bls12_381_g1"]):
            items += [good, (bls.compress(pt), z, y, pi), (c, z, y, bls.compress(pt))]
            want += [0, 3, 3]
        items.append(good)
        want.append(0)
        res, st = ctx.kzg_verify_proof_batch(g2, b"".join(it[0] for it in items), b"".join(it[1].to_bytes(32, "big") for it in items),
                                             b"".join(it[2].to_bytes(32, "big") for it in items), b"".join(it[3] for it in items))
        assert st == want
        assert res == [int(w == 0) for w in want]
    finally:
        ctx.bases_free(g2)


def test_bn254_pairing_rejects_every_component(ctx, cases):
    """pairing_miller: a G2 point of each component order gives status 3; valid neighbours intact"""
    g1, g2 = pyref.G1_GEN, pyref.G2_GEN
    valid = pyref.g1_to_be(g1) + pyref.g2_to_be(g2) + pyref.g1_to_be(pyref.g1_mul(pyref.R - 1, g1)) + pyref.g2_to_be(g2)
    checks = []
    for _, pt in _off(cases["bn254_g2"]):
        checks += [valid, valid + pyref.g1_to_be(g1) + pyref.g2_to_be(pt), pyref.g1_to_be(None) + pyref.g2_to_be(pt)]
    checks.append(valid)
    res, st = ctx.bn254_pairing_check_batch(checks)
    n = (len(checks) - 1) // 3
    assert st == [0, 3, 3] * n + [0]
    assert res == [1, 0, 0] * n + [1]
