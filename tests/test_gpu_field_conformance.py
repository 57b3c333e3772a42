"""Every field and curve primitive on the device against Python integers, at the limb edges where carries go wrong.

tests/csrc/field_conformance.cu runs one primitive per thread over raw limbs (built by ethrex_b200/csrc/Makefile with the
library's own nvcc flags); tests/field_conformance_ref.py holds the integer model, the edge values and the documented
domain of each op.  Field ops compare bit for bit: binary ops over the full cross product of their edges plus 2^16 random
pairs, wider ops over edge tuples plus 2^16 random tuples, exponentiations over their edges plus 2^12 random inputs.  Curve formulas compare with affine arithmetic, with the
accumulators held in non-normalised XYZZ form (lam^2 x, lam^3 y, lam^2, lam^3) so that the exceptional branches compare
different representations of one point.  A failure names the type, the op and the inputs in hex."""
import ctypes
import itertools
import os
import random

import numpy as np
import pytest

import field_conformance_ref as ref

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "build", "libb200zk_conformance.so")
N_RANDOM = 1 << 16
# exponentiations (inv, pow, sqrt) are square-and-multiply chains of the products tested above: 2^12 random inputs, and
# 2^10 over Fp2, where the Python model itself is a square-and-multiply per item
N_RANDOM_EXP = 1 << 12
N_RANDOM_SLOW = 1 << 10


@pytest.fixture(scope="module")
def harness():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    assert os.path.exists(LIB), f"{LIB} is missing: run __graft_entry__.build() first"
    torch.cuda.set_device(0)
    lib = ctypes.CDLL(LIB)
    fn = lib.b200zk_conformance_run
    fn.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint64]
    fn.restype = ctypes.c_int

    def run(tid, op, cols, out_words):
        """cols: uint32 arrays (n, w_k), operand k at word sum(w_<k) of an item; returns uint32 (n, out_words)"""
        arr = np.ascontiguousarray(np.concatenate(cols, axis=1), dtype=np.uint32)
        n, iw = arr.shape
        d_in = torch.from_numpy(arr.view(np.int32)).cuda()
        d_out = torch.zeros((n, out_words), dtype=torch.int32, device="cuda")
        rc = fn(tid, op, d_in.data_ptr(), iw, d_out.data_ptr(), out_words, n)
        assert rc == 0, f"b200zk_conformance_run(type {tid}, op {op}) returned {rc}"
        return d_out.cpu().numpy().view(np.uint32)
    return run


def hexs(x):
    if isinstance(x, tuple):
        return "(" + ", ".join(hexs(c) for c in x) + ")"
    return hex(x)


def assert_all_equal(what, inputs, got, exp):
    bad = [i for i, (g, e) in enumerate(zip(got, exp)) if g != e]
    if bad:
        lines = [f"  inputs {', '.join(hexs(x) for x in inputs[i])}: got {hexs(got[i])}, expected {hexs(exp[i])}" for i in bad[:5]]
        raise AssertionError(f"{what}: {len(bad)} of {len(exp)} results differ\n" + "\n".join(lines))


# ---- inputs -------------------------------------------------------------------------------------------------------------
def field_inputs(F, op, rng):
    """operand tuples over the op's documented domain: the edges' cross product (binary ops), edge tuples (wider ops),
    then random tuples"""
    arity = ref.ARITY[op]
    bound = ref.domain(F, op)
    quad = isinstance(F, ref.Quad)
    E = ref.quad_edges(F) if quad else ref.edges(F, bound)
    slow = quad and op in ("pow", "sqrt")
    n_rand = N_RANDOM_SLOW if slow else N_RANDOM_EXP if op in ("inv", "pow", "sqrt") else N_RANDOM
    if op == "pow":
        es = ref.exponent_edges(F)
        base = E if not slow else E[::4]
        items = [(a, e) for a in base for e in es]
        rb = ref.random_elem(rng, F, bound, n_rand)
        lim = 32 * (F.base.limbs if quad else F.limbs)
        return items + [(a, rng.getrandbits(lim)) for a in rb]
    if op == "scale":
        ks = ref.edges(F.base)
        items = [(a, k) for a in E for k in ks]
        return items + list(zip(ref.random_elem(rng, F, bound, n_rand), ref.random_raw(rng, F.base, F.m, n_rand)))
    if op == "sqrt" and quad:
        return [(a,) for a in fp2_sqrt_inputs(F, rng)]
    if arity == 1:
        return [(a,) for a in E] + [(a,) for a in ref.random_elem(rng, F, bound, n_rand)]
    if arity == 2:
        items = list(itertools.product(E, E))
    else:
        items = [((x, y) * (arity // 2)) for x, y in itertools.product(E, E)]
        items += [((x, y, y, x) * (arity // 4)) for x, y in itertools.product(E[:16], E[:16])]
        top = (F.m - 1, F.m - 1) if quad else F.m - 1
        items.append((top,) * arity)  # the documented worst case of mul4_add: (p - 1)^2 four times
        items += [tuple(rng.choice(E) for _ in range(arity)) for _ in range(n_rand // 4)]
    cols = [ref.random_elem(rng, F, bound, n_rand) for _ in range(arity)]
    return items + list(zip(*cols))


def fp2_sqrt_inputs(F, rng):
    """0; (n, 0) with n a non-residue of Fp (the alpha == -1 branch); (s, 0) with s a residue; (0, t); squares; random"""
    p = F.m
    is_res = lambda v: pow(v, (p - 1) // 2, p) == 1
    non_res = [p - 1, p - 4] + [v for v in (rng.randrange(1, p) for _ in range(64)) if not is_res(v)][:24]
    res = [1, 4] + [v * v % p for v in (rng.randrange(1, p) for _ in range(24))]
    sem = [(0, 0)] + [(v, 0) for v in non_res] + [(v, 0) for v in res]
    sem += [(0, v) for v in [1, p - 1] + [rng.randrange(1, p) for _ in range(24)]]
    sem += [F.mul(a, a) for a in ((rng.randrange(p), rng.randrange(p)) for _ in range(N_RANDOM_SLOW // 2))]
    sem += [(rng.randrange(p), rng.randrange(p)) for _ in range(N_RANDOM_SLOW // 2)]
    assert any(not is_res(v) for v, _ in sem[1:30])
    return [F.enc(a) for a in sem]


def operand_cols(F, op, items):
    arity = ref.ARITY[op]
    cols = []
    for k in range(arity):
        vals = [it[k] for it in items]
        if op == "pow" and k == 1:
            cols.append(ref.pack_ints(vals, F.words))  # the exponent: the operand's slot, low limbs first
        elif op == "scale" and k == 1:
            cols.append(ref.pack_elems(F.base, vals))
        else:
            cols.append(ref.pack_elems(F, vals))
    return cols


FIELD_CASES = [(F, op) for F in ref.PRIMES + ref.QUADS for op in ref.TYPE_OPS[F.name]]


@pytest.mark.parametrize("F,op", FIELD_CASES, ids=[f"{F.name}-{op}" for F, op in FIELD_CASES])
def test_field_op(harness, F, op):
    rng = random.Random(f"{F.name}/{op}")
    items = field_inputs(F, op, rng)
    bound = ref.domain(F, op)
    for it in items:  # every operand inside the op's documented domain
        for k, x in enumerate(it):
            if not ((op == "pow" and k == 1) or (op == "scale" and k == 1)):
                assert all(c < bound for c in F.flat(x))
    secp_sqrt = F is ref.SECP_FP and op == "sqrt"
    out_words = 1 if op == "less" else F.words + (1 if secp_sqrt else 0)
    out = harness(F.tid, ref.OP[op], operand_cols(F, op, items), out_words)
    exp = [ref.expect(F, op, it) for it in items]
    if op == "less":
        got = [int(v) for v in out[:, 0]]
    elif secp_sqrt:
        got = list(zip(ref.unpack_ints(out[:, :8]), (int(v) for v in out[:, 8])))
        got_sq = sum(ok for _, ok in got)
        assert len(items) // 4 < got_sq < 3 * len(items) // 4  # about half the inputs are squares
    else:
        got = ref.unpack_elems(F, out)
    assert_all_equal(f"{F.name} {op}", items, got, exp)
    if op == "sqrt" and isinstance(F, ref.Quad):  # the property the callers rely on: r^2 == a exactly for the squares
        for (a,), r in zip(items, got):
            av = F.dec(a)
            is_square = av == (0, 0) or pow((av[0] ** 2 + av[1] ** 2) % F.m, (F.m - 1) // 2, F.m) == 1  # its norm is a square
            assert (F.mul(F.dec(r), F.dec(r)) == av) == is_square, f"{F.name} sqrt_candidate {hexs(a)} -> {hexs(r)}"


# ---- byte formats -------------------------------------------------------------------------------------------------------
def test_bytes_be48_round_trip(harness):
    rng = random.Random(48)
    p = ref.FP381.m
    vals = ref.edges(ref.FP381) + [p, p + 1, (1 << 384) - 1, 1 << 381, (1 << 381) - 1] + [rng.getrandbits(384) for _ in range(4096)]
    raw = ref.pack_ints(vals, 12)
    stored = harness(ref.T_BYTES, ref.BYTE_OP["store_be48"], [raw], 12)
    assert [stored[i].tobytes() for i in range(len(vals))] == [v.to_bytes(48, "big") for v in vals]
    be = np.frombuffer(b"".join(v.to_bytes(48, "big") for v in vals), dtype=np.uint32).reshape(len(vals), 12)
    assert ref.unpack_ints(harness(ref.T_BYTES, ref.BYTE_OP["load_be48"], [be], 12)) == vals
    masked = ref.unpack_ints(harness(ref.T_BYTES, ref.BYTE_OP["load_be48_masked"], [be], 12))
    assert masked == [v & ((1 << 381) - 1) for v in vals]  # the compressed form's three flag bits cleared
    assert ref.unpack_ints(harness(ref.T_BYTES, ref.BYTE_OP["load_be48"], [stored], 12)) == vals


def test_bytes_fp64_boundary(harness):
    rng = random.Random(64)
    p = ref.FP381.m
    vals = [0, 1, p - 1, p, p + 1, (1 << 384) - 1, 1 << 383] + [rng.randrange(p) for _ in range(1024)]
    items = [(bytes(16), v) for v in vals]
    for k in range(16):  # a nonzero padding byte anywhere, with a value that would be accepted
        items += [(bytes(k) + bytes([1]) + bytes(15 - k), p - 1), (bytes(k) + b"\x80" + bytes(15 - k), 0)]
    src = np.frombuffer(b"".join(pad + v.to_bytes(48, "big") for pad, v in items), dtype=np.uint32).reshape(len(items), 16)
    out = harness(ref.T_BYTES, ref.BYTE_OP["load_fp64"], [src], 13)
    assert ref.unpack_ints(out[:, :12]) == [v for _, v in items]
    ok = [int(x) for x in out[:, 12]]
    assert ok == [int(pad == bytes(16) and v < p) for pad, v in items]
    assert ok[2] == 1 and ok[3] == 0  # p - 1 accepted, p rejected


def test_bytes_be32_and_be256(harness):
    rng = random.Random(32)
    vals = ref.edges(ref.FR381) + ref.edges(ref.SECP_FP) + [(1 << 256) - 1, ref.FR381.m] + [rng.getrandbits(256) for _ in range(4096)]
    be = np.frombuffer(b"".join(v.to_bytes(32, "big") for v in vals), dtype=np.uint32).reshape(len(vals), 8)
    assert ref.unpack_ints(harness(ref.T_BYTES, ref.BYTE_OP["load_be32"], [be], 8)) == vals
    assert ref.unpack_ints(harness(ref.T_BYTES, ref.BYTE_OP["load_be256"], [be], 8)) == vals
    stored = harness(ref.T_BYTES, ref.BYTE_OP["store_be256"], [ref.pack_ints(vals, 8)], 8)
    assert [stored[i].tobytes() for i in range(len(vals))] == [v.to_bytes(32, "big") for v in vals]


# ---- curve formulas -----------------------------------------------------------------------------------------------------
def curve_points(C, rng):
    """G, two random multiples of G and the negation of one: the pairs of these reach P + P, P + (-P) and P + Q"""
    F = C.F
    p1 = C.mul(rng.randrange(2, C.order), C.gen)
    p2 = C.mul(rng.randrange(2, C.order), C.gen)
    pts = [C.gen, p1, C.neg(p1), p2]
    assert all(C.on_curve(q) for q in pts)
    lam = rng.randrange(2, F.m) if F is not ref.FP2_381 and F is not ref.FQ2 else (rng.randrange(F.m), rng.randrange(1, F.m))
    minus_one = F.neg(F.one)
    two = F.add(F.one, F.one)
    return pts, [F.one, lam, minus_one, two]


def xyzz_cols(C, reps):
    F = C.F
    return [ref.pack_elems(F, [F.enc(c[k]) for c in reps]) for k in range(4)]


def affine_cols(C, pts):
    F = C.F
    zero = F.enc(F.zero)
    return [ref.pack_elems(F, [zero if q is None else F.enc(q[k]) for q in pts]) for k in range(2)]


def check_xyzz(C, what, inputs, out, expected):
    """each output is canonical and stands for the expected affine point (ZZ = 0 exactly for the identity)"""
    F = C.F
    quads = [ref.unpack_elems(F, out[:, k * F.words:(k + 1) * F.words]) for k in range(4)]
    got_raw = list(zip(*quads))
    assert all(F.canonical(c) for g in got_raw for c in g), f"{C.name} {what}: a coordinate is not fully reduced"
    got = [C.xyzz_point(tuple(F.dec(c) for c in g)) for g in got_raw]
    assert_all_equal(f"{C.name} {what}", inputs, got, expected)


@pytest.mark.parametrize("C", ref.CURVES, ids=[C.name for C in ref.CURVES])
def test_curve_add(harness, C):
    rng = random.Random(f"{C.name}/add")
    pts, lams = curve_points(C, rng)
    pts = [None] + pts
    acc, q, inputs, exp = [], [], [], []
    for a, b in itertools.product(pts, pts):
        for la, lb in [(lams[0], lams[0]), (lams[1], lams[0]), (lams[0], lams[1]), (lams[1], lams[3]), (lams[2], lams[1])]:
            acc.append(C.xyzz(a, la)); q.append(C.xyzz(b, lb))
            inputs.append((a, b, la, lb)); exp.append(C.add(a, b))
    assert any(a is not None and a == b for a, b, _, _ in inputs) and any(C.add(a, b) is None and a is not None for a, b, _, _ in inputs)
    out = harness(C.tid, ref.CURVE_OP["add"], xyzz_cols(C, acc) + xyzz_cols(C, q), 4 * C.F.words)
    check_xyzz(C, "xyzz_add", inputs, out, exp)


@pytest.mark.parametrize("C", ref.CURVES, ids=[C.name for C in ref.CURVES])
def test_curve_add_mixed(harness, C):
    rng = random.Random(f"{C.name}/add_mixed")
    pts, lams = curve_points(C, rng)
    pts = [None] + pts
    acc, q, inputs, exp = [], [], [], []
    for a, b in itertools.product(pts, pts):
        for la in lams:
            acc.append(C.xyzz(a, la)); q.append(b)
            inputs.append((a, b, la)); exp.append(C.add(a, b))
    out = harness(C.tid, ref.CURVE_OP["add_mixed"], xyzz_cols(C, acc) + affine_cols(C, q), 4 * C.F.words)
    check_xyzz(C, "xyzz_add_mixed", inputs, out, exp)


@pytest.mark.parametrize("C", ref.CURVES, ids=[C.name for C in ref.CURVES])
def test_curve_dbl_mdbl_to_affine(harness, C):
    rng = random.Random(f"{C.name}/dbl")
    F = C.F
    pts, lams = curve_points(C, rng)
    reps = [(a, la) for a in [None] + pts for la in lams]
    inputs = reps
    out = harness(C.tid, ref.CURVE_OP["dbl"], xyzz_cols(C, [C.xyzz(a, la) for a, la in reps]), 4 * F.words)
    check_xyzz(C, "xyzz_dbl", inputs, out, [C.add(a, a) for a, _ in reps])
    out = harness(C.tid, ref.CURVE_OP["mdbl"], affine_cols(C, pts), 4 * F.words)
    check_xyzz(C, "xyzz_mdbl", [(a,) for a in pts], out, [C.add(a, a) for a in pts])
    # to_affine is bit exact: canonical Montgomery coordinates, (0, 0) for the identity
    out = harness(C.tid, ref.CURVE_OP["to_affine"], xyzz_cols(C, [C.xyzz(a, la) for a, la in reps]), 2 * F.words)
    got = list(zip(ref.unpack_elems(F, out[:, :F.words]), ref.unpack_elems(F, out[:, F.words:])))
    zero = F.enc(F.zero)
    assert_all_equal(f"{C.name} xyzz_to_affine", inputs, got, [(zero, zero) if a is None else (F.enc(a[0]), F.enc(a[1])) for a, _ in reps])


@pytest.mark.parametrize("C", ref.CURVES, ids=[C.name for C in ref.CURVES])
def test_curve_scalar_mul(harness, C):
    rng = random.Random(f"{C.name}/scalar_mul")
    pts, _ = curve_points(C, rng)
    r = C.order
    ks = [0, 1, 2, r - 1, r, r + 1, (1 << 256) - 1]
    items = [(q, k) for q in pts[:2] for k in ks]
    out = harness(C.tid, ref.CURVE_OP["scalar_mul"], affine_cols(C, [q for q, _ in items]) + [ref.pack_ints([k for _, k in items], 8)],
                  4 * C.F.words)
    check_xyzz(C, "xyzz_scalar_mul", items, out, [C.mul(k, q) for q, k in items])


@pytest.mark.parametrize("C", ref.CURVES, ids=[C.name for C in ref.CURVES])
def test_curve_on_curve(harness, C):
    rng = random.Random(f"{C.name}/on_curve")
    F = C.F
    pts, _ = curve_points(C, rng)
    off = [(q[0], F.add(q[1], F.one)) for q in pts]  # (x, y + 1)
    items = pts + [None] + off
    out = harness(C.tid, ref.CURVE_OP["on_curve"], affine_cols(C, items), 1)
    assert [int(v) for v in out[:, 0]] == [1] * (len(pts) + 1) + [0] * len(off)
