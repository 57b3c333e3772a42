"""CPU checks of the field-conformance suite itself (tests/test_gpu_field_conformance.py): its edge values lie inside each
op's documented domain, are distinct and cover every limb boundary; its integer model agrees with independent formulas
and with the other references; and the device harness tests/csrc/field_conformance.cu compiles for sm_90a with the
op ids the model uses."""
import os
import random
import re
import subprocess

import pytest

import bls_pairing_ref
import field_conformance_ref as ref
import pyref

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "ethrex_b200", "csrc")
HARNESS = os.path.join(HERE, "csrc", "field_conformance.cu")
ALL = ref.PRIMES + ref.QUADS
CASES = [(F, op) for F in ALL for op in ref.TYPE_OPS[F.name]]
IDS = [f"{F.name}-{op}" for F, op in CASES]


def limb(v, i):
    return (v >> (32 * i)) & 0xffffffff


@pytest.mark.parametrize("F,op", CASES, ids=IDS)
def test_edges_inside_domain_distinct_and_cover_limbs(F, op):
    bound = ref.domain(F, op)
    if isinstance(F, ref.Quad):
        es = ref.quad_edges(F)
        assert len(set(es)) == len(es)
        assert all(c < F.m for e in es for c in e)
        comps = {c for e in es for c in e}
        base = F.base
    else:
        es = ref.edges(F, bound)
        assert len(set(es)) == len(es) and all(0 <= e < bound for e in es)
        comps, base = set(es), F
    m, L = base.m, base.limbs
    R = 1 << (32 * L)
    must = {0, 1, 2, m - 1, m - 2, (m - 1) // 2, (m + 1) // 2, R % m, pow(R, -1, m), m - R % m}
    must |= {pow(2, k, m) for j in range(1, L + 1) for k in (32 * j - 1, 32 * j)}  # every limb boundary
    assert must <= comps
    for i in range(L - 1):  # every limb below the top one is all ones, zero under a nonzero limb above, and top-bit set somewhere
        assert any(limb(v, i) == 0xffffffff for v in comps), i
        assert any(limb(v, i) == 0 and v >> (32 * (i + 1)) for v in comps), i
        assert any(limb(v, i) >> 31 and limb(v, i) != 0xffffffff for v in comps), i
    if bound > m:  # the ops documented for more than canonical inputs get values above m
        above = [e for e in es if e >= m]
        assert len(above) >= 6 and {m, bound - 1} <= set(above)


def test_domains_follow_the_header_comments():
    assert ref.domain(ref.FQ, "mul") == 2 * ref.FQ.m and ref.domain(ref.FR, "mul") == 2 * ref.FR.m
    assert ref.domain(ref.FQ, "sqr") == 1 << 254 > ref.FQ.m  # sqr's comment: a < 2^254
    assert ref.domain(ref.FQ, "mul4_add") == ref.FQ.m and ref.domain(ref.FP381, "mul") == ref.FP381.m
    assert ref.domain(ref.SECP_FP, "mul") == 1 << 256 and ref.domain(ref.SECP_FP, "add") == ref.SECP_FP.m
    assert ref.domain(ref.FP381, "less") == 1 << 384


@pytest.mark.parametrize("F", ref.PRIMES, ids=[F.name for F in ref.PRIMES])
def test_prime_model_against_formulas(F):
    rng = random.Random(F.name)
    m, R = F.m, F.R
    Rinv = pow(R, -1, m)
    xs = ref.edges(F) + [rng.randrange(m) for _ in range(200)]
    for x, y in zip(xs, xs[1:] + xs[:1]):
        assert ref.expect(F, "from_mont", (ref.expect(F, "to_mont", (x,)),)) == x
        assert ref.expect(F, "mul", (x, y)) == x * y * Rinv % m
        assert ref.expect(F, "sqr", (x,)) == x * x * Rinv % m
        assert ref.expect(F, "add", (x, y)) == (x + y) % m and ref.expect(F, "sub", (x, y)) == (x - y) % m
        assert ref.expect(F, "neg", (x,)) == (m - x) % m
        inv = ref.expect(F, "inv", (x,))
        assert ref.expect(F, "mul", (x, inv)) == (R % m if x else 0)  # x inv(x) = the Montgomery one
        assert ref.expect(F, "pow", (x, m - 2)) == inv  # Fermat, as the device computes it
    for x in xs[:20]:
        assert ref.expect(F, "pow", (x, 0)) == R % m
        assert ref.expect(F, "pow", (x, 1)) == x
    if F in (ref.FQ, ref.FR):
        w = m - 1
        assert ref.expect(F, "mul4_add", (w,) * 8) == 4 * w * w * Rinv % m
        assert ref.expect(F, "mul2_add", (1, 2, 3, 4)) == 14 * Rinv % m


def test_sqrt_models():
    p = ref.FP381.m
    rng = random.Random(5)
    for _ in range(50):
        s = rng.randrange(p)
        a = ref.FP381.enc(s * s % p)
        r = ref.FP381.dec(ref.expect(ref.FP381, "sqrt", (a,)))
        assert r * r % p == s * s % p
    q = ref.SECP_FP.m
    assert ref.expect(ref.SECP_FP, "sqrt", (4,))[1] == 1 and ref.expect(ref.SECP_FP, "sqrt", (q - 1,))[1] == 0
    F = ref.FP2_381
    for a in [(p - 1, 0), (p - 4, 0), (4, 0), (0, 1), (0, 5), (3, 7)] + [F.mul(v, v) for v in ((rng.randrange(p), rng.randrange(p)) for _ in range(20))]:
        r = ref.fp2_sqrt_candidate(F, a)
        ok = bls_pairing_ref.f2_sqrt(a)
        assert (F.mul(r, r) == a) == (ok is not None)
        if ok is not None:
            assert r in (ok, F.neg(ok))


def test_quad_model_against_references():
    rng = random.Random(2)
    for F, f2_mul, f2_inv in [(ref.FQ2, pyref.f2_mul, pyref.f2_inv), (ref.FP2_381, bls_pairing_ref.f2_mul, bls_pairing_ref.f2_inv)]:
        m = F.m
        for _ in range(100):
            a, b = (rng.randrange(m), rng.randrange(m)), (rng.randrange(m), rng.randrange(m))
            ra, rb = F.enc(a), F.enc(b)
            assert F.dec(ref.expect(F, "mul", (ra, rb))) == f2_mul(a, b)
            assert F.dec(ref.expect(F, "inv", (ra,))) == f2_inv(a)
            assert F.dec(ref.expect(F, "mul2_sub", (ra, rb, rb, ra))) == (0, 0)
        assert ref.expect(F, "inv", ((0, 0),)) == (0, 0)
    F = ref.FP2_381
    a = (rng.randrange(F.m), rng.randrange(F.m))
    assert F.dec(ref.expect(F, "pow", (F.enc(a), 5))) == bls_pairing_ref.f2_pow(a, 5)
    assert F.dec(ref.expect(F, "mul_xi", (F.enc(a),))) == bls_pairing_ref.f2_mul(a, (1, 1))


def test_limb_packing_round_trip():
    vals = [0, 1, (1 << 384) - 1, ref.FP381.m, 0x0123456789abcdef << 200]
    arr = ref.pack_ints(vals, 12)
    assert arr.shape == (5, 12) and int(arr[2, 11]) == 0xffffffff and int(arr[1, 0]) == 1
    assert ref.unpack_ints(arr) == vals
    F = ref.FP2_381
    elems = [(1, 2), (F.m - 1, 0)]
    assert ref.unpack_elems(F, ref.pack_elems(F, elems)) == elems


@pytest.mark.parametrize("C", ref.CURVES, ids=[C.name for C in ref.CURVES])
def test_curve_model(C):
    G = C.gen
    assert C.on_curve(G) and not C.on_curve((G[0], C.F.add(G[1], C.F.one)))
    assert C.mul(C.order - 1, G) == C.neg(G) and C.add(G, C.neg(G)) is None
    assert C.add(C.add(G, G), G) == C.mul(3, G)
    lam = (5, 3) if isinstance(C.F, ref.Quad) else 5
    assert C.xyzz_point(C.xyzz(G, lam)) == G and C.xyzz_point(C.xyzz(None, lam)) is None


def _enum(src, first):
    m = re.search(r"enum : int \{ " + first + r" = 0,([^}]*)\}", src)
    assert m, first
    return [first] + [re.sub(r"\s*=.*", "", t).strip() for t in m.group(1).split(",") if t.strip()]


def test_harness_ids_match_model():
    src = open(HARNESS).read()
    ops = _enum(src, "ADD")
    assert [o.lower() for o in ops[:-1]] == ref.OPS and ops[-1] == "N_FIELD_OPS"
    assert [o.lower() for o in _enum(src, "LOAD_BE48")[:-1]] == ref.BYTE_OPS
    assert [o[2:].lower() for o in _enum(src, "C_ADD")[:-1]] == ref.CURVE_OPS
    for name in ["T_FQ", "T_FR", "T_FQ2", "T_FP381", "T_FR381", "T_FP2_381", "T_SECP_FP", "T_SECP_FN", "T_BYTES", "T_BN_G1",
                 "T_BN_G2", "T_BLS_G1", "T_BLS_G2", "T_SECP_G"]:
        assert re.search(rf"\b{name} = {getattr(ref, name)}\b", src), name


def test_harness_compiles_for_sm90a(tmp_path):
    """build() leaves tests/build/libb200zk_conformance.so; without it, the same make rule builds one into a temporary
    directory.  Either way the library must hold sm_90a code and export the launcher."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    lib = os.path.join(HERE, "build", "libb200zk_conformance.so")
    if not os.path.exists(lib):
        subprocess.check_call(["make", "-C", CSRC, "-s", "conformance", f"CONF_DIR={tmp_path}"])
        lib = str(tmp_path / "libb200zk_conformance.so")
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    elf = subprocess.run([cuobjdump, "--list-elf", lib], capture_output=True, text=True, check=True).stdout
    assert "sm_90a" in elf
    syms = subprocess.run(["nm", "-D", "--defined-only", lib], capture_output=True, text=True, check=True).stdout
    assert re.search(r"\bT b200zk_conformance_run\b", syms)
