"""Integer model of the device's field and curve primitives -- TEST INFRASTRUCTURE ONLY.

Shared by tests/test_gpu_field_conformance.py (the device harness tests/csrc/field_conformance.cu against it) and
tests/test_field_conformance_host.py (the model against independent formulas).  Every value here is a plain Python
integer.  A field element travels as its raw limbs: x stands for x R^-1 mod m in a Montgomery field (R = 2^(32 limbs)),
so the expected raw result of mul(x, y) is x y R^-1 mod m, whatever the limb pattern of x and y.

The edge values live in raw limb space, where the carries are: 0, 1, 2, m - 1, m - 2, (m -+ 1)/2, R mod m, R^-1 mod m,
m - (R mod m), R^2 mod m, 2^k mod m at every limb boundary, the largest values below a bound whose low limbs are all
ones, alternating 0 / 0xffffffff limbs, every limb's top bit set, and for the ops that accept more than m the same
patterns up to that bound.  Each op is tested over exactly the domain its comment in the header documents (DOMAIN)."""
import numpy as np

import bls_pairing_ref
import bls_ref
import pyref
import secp256k1_ref

# ---- ids of tests/csrc/field_conformance.cu ---------------------------------------------------------------------------
T_FQ, T_FR, T_FQ2, T_FP381, T_FR381, T_FP2_381, T_SECP_FP, T_SECP_FN, T_BYTES = range(9)
T_BN_G1, T_BN_G2, T_BLS_G1, T_BLS_G2, T_SECP_G = range(10, 15)
T_BN_FP6, T_BN_FP12, T_BLS_FP6, T_BLS_FP12 = range(15, 19)
OPS = ["add", "sub", "neg", "dbl", "mul", "sqr", "mul2_add", "mul2_sub", "mul4_add", "to_mont", "from_mont", "inv", "pow",
       "less", "sqrt", "conj", "mul_xi", "scale"]
OP = {name: i for i, name in enumerate(OPS)}
BYTE_OPS = ["load_be48", "load_be48_masked", "store_be48", "load_fp64", "load_be32", "load_be256", "store_be256"]
BYTE_OP = {name: i for i, name in enumerate(BYTE_OPS)}
CURVE_OPS = ["add", "add_mixed", "dbl", "mdbl", "to_affine", "scalar_mul", "on_curve"]
CURVE_OP = {name: i for i, name in enumerate(CURVE_OPS)}
TOWER_OPS = ["zero", "one", "add", "sub", "neg", "mul_v", "mul", "sqr", "conj", "inv", "is_one", "mul_01", "mul_1", "mul_014"]
TOWER_OP = {name: i for i, name in enumerate(TOWER_OPS)}
# the operands of each tower op: "x" a tower element, "f2" an element of the quadratic extension under it
TOWER_OPERANDS = {"zero": [], "one": [], "add": ["x", "x"], "sub": ["x", "x"], "neg": ["x"], "mul_v": ["x"], "mul": ["x", "x"],
                  "sqr": ["x"], "conj": ["x"], "inv": ["x"], "is_one": ["x"], "mul_01": ["x", "f2", "f2"], "mul_1": ["x", "f2"],
                  "mul_014": ["x", "f2", "f2", "f2"]}
# operands per op; pow's second operand is an exponent, scale's a base-field element
ARITY = {"add": 2, "sub": 2, "neg": 1, "dbl": 1, "mul": 2, "sqr": 1, "mul2_add": 4, "mul2_sub": 4, "mul4_add": 8, "to_mont": 1,
         "from_mont": 1, "inv": 1, "pow": 2, "less": 2, "sqrt": 1, "conj": 1, "mul_xi": 1, "scale": 2}


# ---- fields -----------------------------------------------------------------------------------------------------------
class Prime:
    """Z/m with `limbs` 32-bit limbs; Montgomery (R = 2^(32 limbs)) unless mont is False (R = 1)."""

    def __init__(self, name, tid, m, limbs, mont=True):
        self.name, self.tid, self.m, self.limbs, self.words = name, tid, m, limbs, limbs
        self.R = 1 << (32 * limbs) if mont else 1
        self.Rinv = pow(self.R, -1, m)
        self.zero, self.one = 0, 1

    # semantic values
    def add(self, a, b): return (a + b) % self.m
    def sub(self, a, b): return (a - b) % self.m
    def neg(self, a): return -a % self.m
    def mul(self, a, b): return a * b % self.m
    def inv(self, a): return pow(a, -1, self.m) if a else 0
    def pow(self, a, e): return pow(a, e, self.m)
    def is_zero(self, a): return a == 0

    # raw limbs <-> semantic values
    def enc(self, v): return v * self.R % self.m
    def dec(self, x): return x * self.Rinv % self.m
    def flat(self, x): return [x]
    def unflat(self, xs): return xs[0]
    def canonical(self, x): return x < self.m


class Quad:
    """base[u] / (u^2 + 1), elements (c0, c1) of raw base limbs; xi is the tower's non-residue, the factor of mul_xi."""

    def __init__(self, name, tid, base, xi):
        self.name, self.tid, self.base, self.xi = name, tid, base, xi
        self.m, self.limbs, self.words = base.m, base.limbs, 2 * base.limbs
        self.zero, self.one = (0, 0), (1, 0)

    def add(self, a, b): return (self.base.add(a[0], b[0]), self.base.add(a[1], b[1]))
    def sub(self, a, b): return (self.base.sub(a[0], b[0]), self.base.sub(a[1], b[1]))
    def neg(self, a): return (self.base.neg(a[0]), self.base.neg(a[1]))
    def mul(self, a, b):
        m = self.m
        return ((a[0] * b[0] - a[1] * b[1]) % m, (a[0] * b[1] + a[1] * b[0]) % m)
    def inv(self, a):
        d = self.base.inv((a[0] * a[0] + a[1] * a[1]) % self.m)
        return (a[0] * d % self.m, -a[1] * d % self.m)
    def pow(self, a, e):
        acc = self.one
        for bit in bin(e)[2:]:
            acc = self.mul(acc, acc)
            if bit == "1":
                acc = self.mul(acc, a)
        return acc
    def is_zero(self, a): return a == (0, 0)

    def enc(self, v): return (self.base.enc(v[0]), self.base.enc(v[1]))
    def dec(self, x): return (self.base.dec(x[0]), self.base.dec(x[1]))
    def flat(self, x): return [x[0], x[1]]
    def unflat(self, xs): return (xs[0], xs[1])
    def canonical(self, x): return x[0] < self.m and x[1] < self.m


FQ = Prime("fq", T_FQ, pyref.P, 8)
FR = Prime("fr", T_FR, pyref.R, 8)
FQ2 = Quad("fq2", T_FQ2, FQ, (9, 1))
FP381 = Prime("fp381", T_FP381, bls_ref.P, 12)
FR381 = Prime("fr381", T_FR381, bls_ref.R, 8)
FP2_381 = Quad("fp2_381", T_FP2_381, FP381, (1, 1))
SECP_FP = Prime("secp_fp", T_SECP_FP, secp256k1_ref.P, 8, mont=False)
SECP_FN = Prime("secp_fn", T_SECP_FN, secp256k1_ref.N, 8)
PRIMES = [FQ, FR, FP381, FR381, SECP_FP, SECP_FN]
QUADS = [FQ2, FP2_381]

# the ops of each type, as the harness implements them
TYPE_OPS = {
    "fq": ["add", "sub", "neg", "dbl", "mul", "sqr", "mul2_add", "mul2_sub", "mul4_add", "to_mont", "from_mont", "inv", "pow"],
    "fq2": ["add", "sub", "neg", "dbl", "mul", "sqr", "mul2_sub", "inv", "mul_xi"],
    "fp381": ["add", "sub", "neg", "dbl", "mul", "sqr", "mul2_sub", "to_mont", "from_mont", "inv", "pow", "less", "sqrt"],
    "fp2_381": ["add", "sub", "neg", "dbl", "conj", "mul", "sqr", "mul_xi", "scale", "mul2_sub", "inv", "pow", "sqrt"],
    "secp_fp": ["add", "sub", "neg", "dbl", "mul", "sqr", "mul2_sub", "inv", "pow", "sqrt"],
    "secp_fn": ["neg", "mul", "to_mont", "from_mont", "inv"],
}
TYPE_OPS["fr"] = TYPE_OPS["fq"]
TYPE_OPS["fr381"] = [o for o in TYPE_OPS["fp381"] if o != "sqrt"]


def domain(F, op):
    """Exclusive upper bound of each raw operand, from the comment on the op in the header: Fe::mul takes inputs < 2p,
    Fe::sqr a < 2^254, FeBig::less and SecpFp's mul / sqr any limbs; everything else fully reduced values."""
    if isinstance(F, Quad):
        return F.m
    if F in (FQ, FR):
        return {"mul": 2 * F.m, "sqr": 1 << 254}.get(op, F.m)
    if F in (FP381, FR381) and op == "less":
        return 1 << (32 * F.limbs)
    if F is SECP_FP and op in ("mul", "sqr"):
        return 1 << 256
    return F.m


def _ones(k):
    return (1 << (32 * k)) - 1


def limb_patterns(bound, limbs):
    """raw values below `bound` built limb by limb: all-ones low limbs, alternating 0 / 0xffffffff, every top bit set"""
    top_shift = 32 * (limbs - 1)
    top_max = (bound - 1) >> top_shift  # the largest top limb a value below the bound can have
    out = []
    for k in range(1, limbs):  # the largest value below the bound whose low k limbs are all ones
        v = ((bound - 1) >> (32 * k) << (32 * k)) | _ones(k)
        out.append(v if v < bound else v - (1 << (32 * k)))
    alt0 = sum(0xffffffff << (64 * k) for k in range((limbs + 1) // 2)) & _ones(limbs)  # limbs 0, 2, 4, .. all ones
    alt1 = (alt0 << 32) & _ones(limbs)
    tops = sum(0x80000000 << (32 * k) for k in range(limbs - 1))  # every limb's top bit below the top limb
    for low in (alt0 & _ones(limbs - 1), alt1 & _ones(limbs - 1), tops):
        out += [low, low | (top_max << top_shift), low | ((top_max >> 1) << top_shift)]
    out += [v for v in (alt0, alt1, tops | (0x80000000 << top_shift)) if v < bound]
    return [v for v in out if v < bound]


def edges(F, bound=None):
    """distinct raw edge values of a prime field below `bound` (default m), canonical ones first"""
    m, L = F.m, F.limbs
    bound = bound or m
    R = 1 << (32 * L)
    vals = [0, 1, 2, m - 1, m - 2, (m - 1) // 2, (m + 1) // 2, R % m, pow(R, -1, m), m - R % m, R * R % m]
    vals += [pow(2, k, m) for j in range(1, L + 1) for k in (32 * j - 1, 32 * j)]
    vals += limb_patterns(m, L)
    if bound > m:  # the ops that take more than canonical values: the same patterns up to their bound
        vals += [m, m + 1, m + 2, bound - 1, bound - 2, m + R % m, m + (m - 1) // 2, m + 0xffffffff, bound - (1 << 32)]
        vals += [v for v in (2 * m - 1, 2 * m - 2) if v < bound]
        vals += [1 << k for j in range(1, L + 1) for k in (32 * j - 1, 32 * j) if m <= (1 << k) < bound]
        vals += limb_patterns(bound, L)
    seen, out = set(), []
    for v in vals:
        if v < bound and v not in seen:
            seen.add(v)
            out.append(v)
    return out


def exponent_edges(F):
    L = F.limbs if not isinstance(F, Quad) else F.base.limbs
    m = F.m
    return [0, 1, 2, 3, m - 1, m - 2, (m + 1) // 4, (m - 1) // 2, _ones(L), 1 << (32 * L - 1), 0xffffffff, 1 << 32,
            _ones(L) ^ 0xffffffff]


def quad_edges(F):
    """Fp2 elements from the base field's edges: (e, 0), (0, e), (e, e), (e, m - 1 - e)"""
    es = edges(F.base)
    out = [(e, 0) for e in es] + [(0, e) for e in es[1:]] + [(e, e) for e in es[1:]] + [(e, F.m - 1 - e) for e in es]
    return list(dict.fromkeys(out))


def random_raw(rng, F, bound, count):
    """half uniform below the bound, half built from structured limbs (0, 1, 0xffffffff, 0x80000000, ...)"""
    L = F.limbs
    top_shift = 32 * (L - 1)
    top_max = (bound - 1) >> top_shift
    picks = [0, 1, 0xffffffff, 0x80000000, 0x7fffffff, 0xfffffffe]
    out = [rng.randrange(bound) for _ in range(count - count // 2)]
    for _ in range(count // 2):
        v = 0
        for k in range(L - 1):
            v |= (rng.choice(picks) if rng.random() < 0.6 else rng.getrandbits(32)) << (32 * k)
        top = rng.choice([0, top_max, top_max >> 1, rng.randrange(top_max + 1)])
        v |= top << top_shift
        out.append(v if v < bound else v % bound)
    return out


def random_elem(rng, F, bound, count):
    if isinstance(F, Quad):
        a, b = random_raw(rng, F.base, F.m, count), random_raw(rng, F.base, F.m, count)
        rng.shuffle(b)
        return list(zip(a, b))
    return random_raw(rng, F, bound, count)


# ---- expected raw results ---------------------------------------------------------------------------------------------
def fp2_sqrt_candidate(F, a):
    """Fp2_381::sqrt_candidate on semantic values: Adj and Rodriguez-Henriquez, Algorithm 9 (p = 3 mod 4)"""
    p = F.m
    a1 = F.pow(a, (p - 3) // 4)
    x0 = F.mul(a1, a)
    alpha = F.mul(a1, x0)
    if alpha == (p - 1, 0):
        return (-x0[1] % p, x0[0])  # u x0
    return F.mul(F.pow(F.add(F.one, alpha), (p - 1) // 2), x0)


def expect(F, op, xs):
    """the raw result of `op` on raw operands xs (an int for LESS, (root, is_square) for SecpFp's sqrt)"""
    if op == "less":
        return int(xs[0] < xs[1])
    if isinstance(F, Prime) and op == "to_mont":
        return xs[0] * F.R % F.m
    if isinstance(F, Prime) and op == "from_mont":
        return xs[0] * F.Rinv % F.m
    if op == "pow":
        return F.enc(F.pow(F.dec(xs[0]), xs[1]))
    if op == "scale":
        k = F.base.dec(xs[1])
        a = F.dec(xs[0])
        return F.enc((a[0] * k % F.m, a[1] * k % F.m))
    v = [F.dec(x) for x in xs]
    if op == "add": r = F.add(v[0], v[1])
    elif op == "sub": r = F.sub(v[0], v[1])
    elif op == "neg": r = F.neg(v[0])
    elif op == "dbl": r = F.add(v[0], v[0])
    elif op == "mul": r = F.mul(v[0], v[1])
    elif op == "sqr": r = F.mul(v[0], v[0])
    elif op == "mul2_add": r = F.add(F.mul(v[0], v[1]), F.mul(v[2], v[3]))
    elif op == "mul2_sub": r = F.sub(F.mul(v[0], v[1]), F.mul(v[2], v[3]))
    elif op == "mul4_add": r = F.add(F.add(F.mul(v[0], v[1]), F.mul(v[2], v[3])), F.add(F.mul(v[4], v[5]), F.mul(v[6], v[7])))
    elif op == "inv": r = F.inv(v[0])
    elif op == "conj": r = (v[0][0], F.base.neg(v[0][1]))
    elif op == "mul_xi": r = F.mul(v[0], F.xi)
    elif op == "sqrt":
        if isinstance(F, Quad):
            r = fp2_sqrt_candidate(F, v[0])
        else:
            root = pow(v[0], (F.m + 1) // 4, F.m)
            if F is SECP_FP:
                return (root, int(root * root % F.m == v[0]))
            r = root
    else:
        raise KeyError(op)
    return F.enc(r)


# ---- the pairing towers ---------------------------------------------------------------------------------------------
class Ext:
    """base[t] / (t^n - nr), elements n-tuples of base elements, products by schoolbook polynomial arithmetic: Fp6 =
    F2[v] / (v^3 - xi) over a Quad, Fp12 = Fp6[w] / (w^2 - v) over that.  `quad` is the F2 at the bottom."""

    def __init__(self, name, tid, base, n, nr):
        self.name, self.tid, self.base, self.n, self.nr = name, tid, base, n, nr
        self.quad = base if isinstance(base, Quad) else base.quad
        self.m, self.limbs, self.words = base.m, base.limbs, n * base.words
        self.zero = (base.zero,) * n
        self.one = (base.one,) + (base.zero,) * (n - 1)

    def add(self, a, b): return tuple(self.base.add(x, y) for x, y in zip(a, b))
    def sub(self, a, b): return tuple(self.base.sub(x, y) for x, y in zip(a, b))
    def neg(self, a): return tuple(self.base.neg(x) for x in a)
    def mul(self, a, b):
        B, n = self.base, self.n
        c = [B.zero] * (2 * n - 1)
        for i in range(n):
            for j in range(n):
                c[i + j] = B.add(c[i + j], B.mul(a[i], b[j]))
        for k in range(2 * n - 2, n - 1, -1):  # t^k = nr t^(k - n)
            c[k - n] = B.add(c[k - n], B.mul(c[k], self.nr))
        return tuple(c[:n])
    def is_zero(self, a): return a == self.zero

    def enc(self, v): return tuple(self.base.enc(x) for x in v)
    def dec(self, x): return tuple(self.base.dec(c) for c in x)
    def flat(self, x): return [w for c in x for w in self.base.flat(c)]
    def unflat(self, xs):
        k = len(xs) // self.n
        return tuple(self.base.unflat(xs[i * k:(i + 1) * k]) for i in range(self.n))
    def canonical(self, x): return all(self.base.canonical(c) for c in x)


def _tower(prefix, tid6, tid12, F2):
    f6 = Ext(prefix + "_fp6", tid6, F2, 3, F2.xi)
    return f6, Ext(prefix + "_fp12", tid12, f6, 2, (F2.zero, F2.one, F2.zero))  # w^2 = v


BN_FP6, BN_FP12 = _tower("bn254", T_BN_FP6, T_BN_FP12, FQ2)
BLS_FP6, BLS_FP12 = _tower("bls12_381", T_BLS_FP6, T_BLS_FP12, FP2_381)
TOWERS = [BN_FP6, BN_FP12, BLS_FP6, BLS_FP12]
TOWER_TYPE_OPS = {6: ["zero", "one", "add", "sub", "neg", "mul_v", "mul", "inv", "mul_01", "mul_1"],
                  12: ["one", "mul", "sqr", "conj", "inv", "is_one", "mul_014"]}


def tower_ops(T):
    return TOWER_TYPE_OPS[6 if T.n == 3 else 12]


def base_coords(T):
    """the number of base-field coordinates of a tower element"""
    return T.words // T.limbs


def tower_edges(T):
    """raw tower elements: zero, one, every base coordinate at one edge of edges(), the edges spread over the coordinates,
    and elements with all but one top-level component zero"""
    P = T.quad.base
    es, k = edges(P), base_coords(T)
    zero = T.unflat([0] * k)
    out = [zero, T.enc(T.one)]
    out += [T.unflat([e] * k) for e in es[1:]]
    out += [T.unflat([es[(i + j) % len(es)] for j in range(k)]) for i in range(len(es))]
    part = k // T.n
    for c in range(T.n):  # component c only, its coordinates at the edges
        for i in range(0, len(es), 4):
            out.append(T.unflat([es[(i + j) % len(es)] if c * part <= j < (c + 1) * part else 0 for j in range(k)]))
    return list(dict.fromkeys(out))


def random_tower(rng, T, count):
    """random raw tower elements: uniform and structured coordinates, a fifth of them with one zero component"""
    P = T.quad.base
    k, part = base_coords(T), base_coords(T) // T.n
    cols = [random_raw(rng, P, P.m, count) for _ in range(k)]
    for c in cols:
        rng.shuffle(c)
    out = []
    for i in range(count):
        coords = [c[i] for c in cols]
        if i % 5 == 0:
            z = rng.randrange(T.n)
            coords[z * part:(z + 1) * part] = [0] * part
        out.append(T.unflat(coords))
    return out


def tower_expect(T, op, xs):
    """the raw result of a tower op on raw operands (an int for is_one); inv has no expected value (see the test)"""
    if op == "zero": return T.enc(T.zero)
    if op == "one": return T.enc(T.one)
    F2 = T.quad
    v = [T.dec(x) if k == "x" else F2.dec(x) for k, x in zip(TOWER_OPERANDS[op], xs)]
    if op == "add": r = T.add(v[0], v[1])
    elif op == "sub": r = T.sub(v[0], v[1])
    elif op == "neg": r = T.neg(v[0])
    elif op == "mul": r = T.mul(v[0], v[1])
    elif op == "sqr": r = T.mul(v[0], v[0])
    elif op == "mul_v": r = T.mul(v[0], (F2.zero, F2.one, F2.zero))
    elif op == "conj": r = (v[0][0], T.base.neg(v[0][1]))
    elif op == "is_one": return int(v[0] == T.one)
    elif op == "mul_01": r = T.mul(v[0], (v[1], v[2], F2.zero))
    elif op == "mul_1": r = T.mul(v[0], (F2.zero, v[1], F2.zero))
    elif op == "mul_014":  # c0 + c1 v + c4 v w
        r = T.mul(v[0], ((v[1], v[2], F2.zero), (F2.zero, v[3], F2.zero)))
    else:
        raise KeyError(op)
    return T.enc(r)


# ---- limbs <-> numpy --------------------------------------------------------------------------------------------------
def pack_ints(vals, words):
    """ints -> uint32 array (len(vals), words), little-endian limbs"""
    return np.frombuffer(b"".join(v.to_bytes(4 * words, "little") for v in vals), dtype="<u4").reshape(len(vals), words).copy()


def unpack_ints(arr):
    """uint32 array (n, words) -> ints"""
    arr = np.ascontiguousarray(arr, dtype="<u4")
    step = 4 * arr.shape[1]
    buf = arr.tobytes()
    return [int.from_bytes(buf[i:i + step], "little") for i in range(0, len(buf), step)]


def pack_elems(F, elems):
    """raw field elements -> uint32 array (n, F.words)"""
    flat = [c for e in elems for c in F.flat(e)]
    return pack_ints(flat, F.limbs).reshape(len(elems), F.words)


def unpack_elems(F, arr):
    comps = F.words // F.limbs
    ints = unpack_ints(np.ascontiguousarray(arr).reshape(-1, F.limbs))
    return [F.unflat(ints[i:i + comps]) for i in range(0, len(ints), comps)]


# ---- curves: affine group law on semantic values, None = identity ------------------------------------------------------
class Curve:
    def __init__(self, name, tid, F, b, order, gen):
        self.name, self.tid, self.F, self.b, self.order, self.gen = name, tid, F, b, order, gen

    def on_curve(self, pt):
        if pt is None:
            return True
        F, (x, y) = self.F, pt
        return F.mul(y, y) == F.add(F.mul(F.mul(x, x), x), self.b)

    def neg(self, pt):
        return None if pt is None else (pt[0], self.F.neg(pt[1]))

    def add(self, a, b):
        F = self.F
        if a is None:
            return b
        if b is None:
            return a
        (x1, y1), (x2, y2) = a, b
        if x1 == x2:
            if y1 != y2 or F.is_zero(y1):
                return None
            xx = F.mul(x1, x1)
            lam = F.mul(F.add(F.add(xx, xx), xx), F.inv(F.add(y1, y1)))
        else:
            lam = F.mul(F.sub(y2, y1), F.inv(F.sub(x2, x1)))
        x3 = F.sub(F.sub(F.mul(lam, lam), x1), x2)
        return (x3, F.sub(F.mul(lam, F.sub(x1, x3)), y1))

    def mul(self, k, pt):
        """k pt for pt in the order-`order` subgroup: double-and-add over k mod order"""
        acc = None
        for bit in bin(k % self.order)[2:]:
            acc = self.add(acc, acc)
            if bit == "1":
                acc = self.add(acc, pt)
        return acc

    def xyzz(self, pt, lam):
        """semantic XYZZ coordinates (lam^2 x, lam^3 y, lam^2, lam^3) of pt; the identity is all zero"""
        F = self.F
        if pt is None:
            return (F.zero,) * 4
        l2 = F.mul(lam, lam)
        l3 = F.mul(l2, lam)
        return (F.mul(l2, pt[0]), F.mul(l3, pt[1]), l2, l3)

    def xyzz_point(self, c):
        """the affine point an XYZZ quadruple stands for, or "bad" when ZZ^3 != ZZZ^2"""
        F = self.F
        x, y, zz, zzz = c
        if F.is_zero(zz):
            return None
        if F.mul(F.mul(zz, zz), zz) != F.mul(zzz, zzz):
            return "bad"
        return (F.mul(x, F.inv(zz)), F.mul(y, F.inv(zzz)))


CURVES = [
    Curve("bn254_g1", T_BN_G1, FQ, 3, pyref.R, pyref.G1_GEN),
    Curve("bn254_g2", T_BN_G2, FQ2, pyref.B_G2, pyref.R, pyref.G2_GEN),
    Curve("bls12_381_g1", T_BLS_G1, FP381, 4, bls_ref.R, bls_ref.G1),
    Curve("bls12_381_g2", T_BLS_G2, FP2_381, bls_pairing_ref.B2, bls_ref.R, bls_pairing_ref.G2),
    Curve("secp256k1", T_SECP_G, SECP_FP, 7, secp256k1_ref.N, secp256k1_ref.G),
]
