"""CPU checks of P-256 verification (P256VERIFY, EIP-7951): the Python oracle (tests/secp256r1_ref.py) against the
`cryptography` package (OpenSSL's P-256) on signatures, tampered items, high-s twins and the constructed edge cases, the
curve constants, and a host build of the device's own __host__ __device__ fields, a = -3 doublings and verification
(ethrex_b200/csrc/secp256r1.cuh, compiled by nvcc into a CPU program) against the oracle.  Finally the ptxas report of the
new kernels against DESIGN.md section 4.11."""
import os
import random
import re
import subprocess

import pytest
from cryptography.exceptions import InvalidSignature
from cryptography.hazmat.primitives import hashes
from cryptography.hazmat.primitives.asymmetric import ec, utils

import secp256r1_ref as ref

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "ethrex_b200", "csrc")
P, N = ref.P, ref.N
R = 2**256


def h32(x: int) -> str:
    return x.to_bytes(32, "big").hex()


def crypto_item(rng) -> bytes:
    """a 160-byte P256VERIFY input signed by OpenSSL over a random 32-byte digest"""
    key = ec.derive_private_key(rng.randrange(1, N), ec.SECP256R1())
    digest = rng.randbytes(32)
    r, s = utils.decode_dss_signature(key.sign(digest, ec.ECDSA(utils.Prehashed(hashes.SHA256()))))
    pub = key.public_key().public_numbers()
    return ref.encode(int.from_bytes(digest, "big"), r, s, (pub.x, pub.y))


def crypto_verify(inp: bytes):
    """OpenSSL's answer, or None when it does not take (qx, qy) as a public key or (r, s) as a signature"""
    h, r, s, qx, qy = ref.decode(inp)
    try:
        key = ec.EllipticCurvePublicNumbers(qx, qy, ec.SECP256R1()).public_key()
        sig = utils.encode_dss_signature(r, s)
    except ValueError:
        return None
    try:
        key.verify(sig, h.to_bytes(32, "big"), ec.ECDSA(utils.Prehashed(hashes.SHA256())))
        return True
    except InvalidSignature:
        return False


def flip(inp: bytes, field: int, bit: int) -> bytes:
    b = bytearray(inp)
    b[32 * field + 31 - bit // 8] ^= 1 << (bit % 8)
    return bytes(b)


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("p256") / "secp256r1_host_check")
    subprocess.check_call([nvcc, "-std=c++17", "-O2", "-o", exe, os.path.join(HERE, "secp256r1_host_check.cu")])

    def run(lines):
        out = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True, timeout=600).stdout
        res = out.splitlines()
        assert len(res) == len(lines)
        return res
    return run


# ---- oracle -----------------------------------------------------------------------------------------------------------------
def test_constants():
    assert ref.on_curve(ref.G)
    assert ref.mul(N, ref.G) is None and ref.mul(N - 1, ref.G) == ref.neg(ref.G)
    assert ref.A == -3 and P % 4 == 3
    # the curve equation the oracle uses is the one OpenSSL's P-256 keys satisfy
    pub = ec.derive_private_key(12345, ec.SECP256R1()).public_key().public_numbers()
    assert ref.mul(12345, ref.G) == (pub.x, pub.y)
    assert (pub.y ** 2 - pub.x ** 3 + 3 * pub.x - ref.B) % P == 0


def test_oracle_against_openssl():
    rng = random.Random(1)
    items = [crypto_item(rng) for _ in range(300)]
    for inp in items:
        assert ref.verify(inp)
        twin = ref.high_s(inp)
        assert ref.verify(twin) and crypto_verify(twin) is True
    for i, inp in enumerate(items):
        field = i % 5
        t = flip(inp, field, rng.randrange(256))
        want = crypto_verify(t)
        got = ref.verify(t)
        assert got is False
        if want is not None:  # OpenSSL refuses off-curve keys and r or s outside [1, n - 1] before it verifies
            assert got == want


@pytest.mark.parametrize("case", ref.constructed_cases(), ids=lambda c: c[0])
def test_constructed_cases(case):
    name, inp, expected = case
    assert ref.verify(inp) == expected
    want = crypto_verify(inp)
    if want is not None:
        assert want == expected, name


def test_constructed_cases_cover_the_edges():
    cases = {name: exp for name, _, exp in ref.constructed_cases()}
    assert cases["x_above_n"] and cases["equal_points_2g"] and not cases["opposite_points"] and not cases["r_prime_infinity"]


# ---- host build of secp256r1.cuh against the oracle ----------------------------------------------------------------------
@pytest.mark.parametrize("prefix,m", [("p", P), ("n", N)])
def test_host_fields(host, prefix, m):
    rng = random.Random(11 if prefix == "p" else 12)
    edges = sorted({0, 1, 2, m - 1, m - 2, 2**224 % m, 2**192 % m, 2**96 - 1, 2**96 + 1, 2**255 % m, R % m, R * R % m,
                    (m - 1) // 2, (m + 1) // 2, 0xFFFFFFFF, 2**128 - 1})
    vals = edges + [rng.randrange(m) for _ in range(3000)]
    ri = pow(R, -1, m)
    lines, exp = [], []
    for a in edges:
        for b in edges:
            lines += [f"{prefix}mul {h32(a)} {h32(b)}", f"{prefix}add {h32(a)} {h32(b)}", f"{prefix}sub {h32(a)} {h32(b)}"]
            exp += [a * b * ri % m, (a + b) % m, (a - b) % m]
        lines.append(f"{prefix}sqr {h32(a)}"); exp.append(a * a * ri % m)
    for a, b in zip(vals, vals[1:]):
        lines += [f"{prefix}mul {h32(a)} {h32(b)}", f"{prefix}sqr {h32(a)}", f"{prefix}add {h32(a)} {h32(b)}", f"{prefix}sub {h32(a)} {h32(b)}"]
        exp += [a * b * ri % m, a * a * ri % m, (a + b) % m, (a - b) % m]
    for a in edges + vals[len(edges):len(edges) + 300]:
        lines.append(f"{prefix}inv {h32(a)}"); exp.append(pow(a, m - 2, m))
    assert host(lines) == [h32(e) for e in exp]


def test_host_montgomery_round_trip(host):
    rng = random.Random(13)
    vals = [0, 1, P - 1, 2**224, 2**192, 2**96 + 1] + [rng.randrange(P) for _ in range(200)]
    res = host([f"mont {h32(a)}" for a in vals] + [f"unmont {h32(a * R % P)}" for a in vals])
    assert res == [h32(a * R % P) for a in vals] + [h32(a) for a in vals]


def test_host_a_minus_3_doublings(host):
    rng = random.Random(14)
    pts = [ref.G, ref.mul(2, ref.G), next(ref.lift_x(x) for x in range(1, 1000) if ref.lift_x(x) is not None)]
    pts += [ref.mul(rng.randrange(1, N), ref.G) for _ in range(60)]
    lams = [1, 2, N - 1, P - 1] + [rng.randrange(1, P) for _ in range(3)]
    lines, exp = [], []
    for i, (x, y) in enumerate(pts):
        d = ref.add((x, y), (x, y))
        lam = lams[i % len(lams)]
        lines += [f"mdbl {h32(x)} {h32(y)}", f"dbl {h32(x)} {h32(y)} {h32(lam)}", f"add {h32(x)} {h32(y)} {h32(x)} {h32(y)} {h32(lam)}",
                  f"add {h32(x)} {h32(y)} {h32(x)} {h32(P - y)} {h32(lam)}", f"oncurve {h32(x)} {h32(y)}", f"oncurve {h32(x)} {h32((y + 1) % P)}"]
        exp += [f"{h32(d[0])} {h32(d[1])}"] * 3 + ["inf", "1", "0"]
    assert host(lines) == exp


def test_host_g_table_entries(host):
    ds = [1, 2, 3, 4094, 4095]
    assert host([f"gmul {d}" for d in ds]) == ["%s %s" % (h32(q[0]), h32(q[1])) for q in (ref.mul(d, ref.G) for d in ds)]


def test_host_verify(host):
    rng = random.Random(19)
    items = [inp for _, inp, _ in ref.constructed_cases()]
    for i in range(300):
        priv, h = rng.randrange(1, N), rng.randrange(R)
        r, s = ref.sign(priv, h, rng.randrange(1, N))
        inp = ref.encode(h, r, s, ref.mul(priv, ref.G))
        items.append(inp if i % 2 == 0 else flip(inp, rng.randrange(5), rng.randrange(256)))
    items += [rng.randbytes(160) for _ in range(100)]
    res = host([f"verify {inp.hex()}" for inp in items])
    want = [ref.verify(inp) for inp in items]
    assert res == ["1" if w else "0" for w in want]
    assert 150 <= sum(want) < 200


# ---- ptxas report ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kernel", ["secp256r1_verify_kernel", "secp256r1_gtab_build"])
def test_ptxas_report_matches_design(kernel):
    log = os.path.join(CSRC, "build", "secp256r1.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("secp256r1.ptxas.log not built")
    m = re.search(r"Function properties for \w*" + kernel + r"\w*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads\nptxas info\s*: Used (\d+) registers", open(log).read())
    assert m, f"no ptxas report for {kernel}"
    stack, stores, loads, regs = map(int, m.groups())
    design = open(os.path.join(ROOT, "DESIGN.md")).read()
    row = re.search(r"^\| `" + kernel + r"` \| (\d+) \| (\d+) \| (\d+) \| (\d+) / (\d+) \|", design, re.M)
    assert row, f"DESIGN.md section 4.11 has no row for {kernel}"
    assert tuple(map(int, row.groups()[1:])) == (regs, stack, stores, loads)
