"""CPU checks of signer recovery on secp256k1: the Python oracle (tests/secp256k1_ref.py) against the `cryptography`
package and the ethrex L1 genesis keys, every status from a constructed input, and a host build of the device's own
__host__ __device__ field, scalar, Keccak and recovery code (ethrex_b200/csrc/secp256k1.cuh, compiled by nvcc into a CPU
program) against the oracle.  Finally the ptxas report of the new kernels against DESIGN.md section 4.10."""
import hashlib
import json
import os
import random
import re
import subprocess

import pytest
from cryptography.hazmat.primitives import hashes
from cryptography.hazmat.primitives.asymmetric import ec, utils

import secp256k1_ref as ref

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "ethrex_b200", "csrc")
P, N = ref.P, ref.N
EMPTY_KECCAK_HASH = "c5d2460186f7233c927e7db2dcc703c0e500b653ca82273b7bfad8045d85a470"  # ethrex EMPTY_KECCACK_HASH


def h32(x: int) -> str:
    return x.to_bytes(32, "big").hex()


def crypto_sign(priv, digest: bytes) -> bytes:
    """a `cryptography` signature over a raw 32-byte digest, as r | s | recid (recid found by the oracle)"""
    key = ec.derive_private_key(priv, ec.SECP256K1())
    r, s = utils.decode_dss_signature(key.sign(digest, ec.ECDSA(utils.Prehashed(hashes.SHA256()))))
    pub = key.public_key().public_numbers()
    for recid in (0, 1):
        sig = r.to_bytes(32, "big") + s.to_bytes(32, "big") + bytes([recid])
        st, q = ref.recover_point(sig, digest)
        if st == ref.OK and q == (pub.x, pub.y):
            return sig
    raise AssertionError("no recid recovers the signer")


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("secp") / "secp256k1_host_check")
    subprocess.check_call([nvcc, "-std=c++17", "-O2", "-o", exe, os.path.join(HERE, "secp256k1_host_check.cu")])

    def run(lines):
        out = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True, timeout=600).stdout
        res = out.splitlines()
        assert len(res) == len(lines)
        return res
    return run


# ---- oracle ---------------------------------------------------------------------------------------------------------------
def test_keccak_oracle():
    assert ref.keccak256(b"").hex() == EMPTY_KECCAK_HASH
    assert ref.keccak256(b"abc").hex() == "4e03657aea45a94fc7d47ba826c8d667c0d1e6e33a64a036ec44f58fa12d6c45"


def test_oracle_recovers_cryptography_signers():
    rng = random.Random(4)
    recids = set()
    for _ in range(24):
        priv = rng.randrange(1, N)
        digest = rng.randbytes(32)
        sig = crypto_sign(priv, digest)
        recids.add(sig[64])
        pub = ec.derive_private_key(priv, ec.SECP256K1()).public_key().public_numbers()
        assert ref.recover(sig, digest) == (ref.OK, ref.address_hash((pub.x, pub.y)))
        assert ref.verify((pub.x, pub.y), sig, digest)
    assert recids == {0, 1}


def test_golden_keys_give_genesis_addresses():
    keys = json.load(open(os.path.join(HERE, "golden", "secp256k1_l1_keys.json")))["keys"]
    assert len(keys) == 192
    assert {"private_key": "bcdf20249abf0ed6d944c0288fad489e33f66b3960d9e6229c1cd214ed3bbe31",
            "address": "8943545177806ed17b9f23f0a21ee5948ecaa776"} in keys
    digest = hashlib.sha256(b"ethrex l1 genesis").digest()
    for k in keys:
        sig = ref.low_s(crypto_sign(int(k["private_key"], 16), digest))
        st, h = ref.recover(sig, digest, low_s=True)
        assert st == ref.OK and h[12:].hex() == k["address"]


@pytest.mark.parametrize("case", ref.status_cases(), ids=lambda c: c[0])
def test_status_cases(case):
    name, sig, msg, low_s, expected = case
    st, q = ref.recover_point(sig, msg, low_s)
    assert st == expected
    if st == ref.OK:
        assert ref.on_curve(q) and ref.verify(q, sig, msg)  # the recovered key verifies the signature it came from
    if name.startswith("recid_2_recovers") or name.startswith("recid_3_recovers"):
        assert int.from_bytes(sig[:32], "big") < P - N


# ---- host build of secp256k1.cuh against the oracle ----------------------------------------------------------------------
def test_host_keccak(host):
    rng = random.Random(7)
    lens = [0, 1, 31, 32, 64, 135, 136, 137, 200, 271, 272, 273, 500, 1000]
    msgs = [rng.randbytes(n) for n in lens]
    lines = [f"sponge 1 {m.hex() or '-'}" for m in msgs] + [f"sponge 6 {m.hex() or '-'}" for m in msgs]
    keys = [rng.randbytes(64) for _ in range(64)] + [bytes(64), b"\xff" * 64]
    lines += [f"keccak64 {k.hex()}" for k in keys]
    res = host(lines)
    k = len(msgs)
    assert res[0] == EMPTY_KECCAK_HASH
    assert res[:k] == [ref.keccak256(m).hex() for m in msgs]
    assert res[k:2 * k] == [hashlib.sha3_256(m).hexdigest() for m in msgs]  # the same permutation under SHA-3's padding
    assert res[2 * k:] == [ref.keccak256(x).hex() for x in keys]


def test_host_base_field(host):
    rng = random.Random(11)
    edges = [0, 1, 2, 977, 2**32 + 977, P - 2, P - 1, 2**255, 2**256 - 2**32 - 978]
    big = [P, P + 1, 2**256 - 1, 2**256 - 2**32]  # >= p: mul and sqr take any 256-bit value
    vals = edges + [rng.randrange(P) for _ in range(2000)]
    lines, exp = [], []
    for a in edges + big:
        for b in edges + big:
            lines.append(f"mul {h32(a)} {h32(b)}"); exp.append(a * b % P)
        lines.append(f"sqr {h32(a)}"); exp.append(a * a % P)
    for i in range(0, len(vals) - 1):
        a, b = vals[i], vals[i + 1]
        lines += [f"mul {h32(a)} {h32(b)}", f"sqr {h32(a)}", f"add {h32(a)} {h32(b)}", f"sub {h32(a)} {h32(b)}"]
        exp += [a * b % P, a * a % P, (a + b) % P, (a - b) % P]
    for a in vals[:300]:
        lines.append(f"inv {h32(a)}"); exp.append(pow(a, P - 2, P))
    res = host(lines)
    assert res == [h32(e) for e in exp]


def test_host_sqrt(host):
    rng = random.Random(13)
    vals = [0, 1, 7, P - 1, P - 7] + [rng.randrange(P) for _ in range(1000)]
    res = host([f"sqrt {h32(a)}" for a in vals])
    for a, r in zip(vals, res):
        root = ref.sqrt(a)
        if root is None:
            assert r == "0", a
        else:
            assert r.startswith("1 ") and pow(int(r[2:], 16), 2, P) == a % P
    assert sum(r == "0" for r in res) > 400  # about half are non-residues


def test_host_scalar_field(host):
    rng = random.Random(17)
    vals = [1, 2, N - 1, N - 2, ref.N_HALF] + [rng.randrange(1, N) for _ in range(1500)]
    lines = [f"ninv {h32(a)}" for a in vals] + [f"nmul {h32(a)} {h32(b)}" for a, b in zip(vals, vals[1:])]
    exp = [pow(a, -1, N) for a in vals] + [a * b % N for a, b in zip(vals, vals[1:])]
    assert host(lines) == [h32(e) for e in exp]


def test_host_recovery(host):
    rng = random.Random(19)
    items = [(sig, msg, low) for _, sig, msg, low, _ in ref.status_cases()]
    for i in range(300):
        digest = rng.randbytes(32)
        sig = ref.sign(rng.randrange(1, N), digest, rng.randrange(1, N))
        items.append((sig, digest, bool(i & 1)))
    for _ in range(100):  # arbitrary bytes: mostly status 0 or 3, and every recid value
        items.append((rng.randbytes(64) + bytes([rng.randrange(6)]), rng.randbytes(32), rng.random() < 0.5))
    res = host([f"recover {int(low)} {sig.hex()} {msg.hex()}" for sig, msg, low in items])
    seen = set()
    for (sig, msg, low), r in zip(items, res):
        st, h = ref.recover(sig, msg, low)
        seen.add(st)
        assert r == f"{st} {h.hex()}", (sig.hex(), msg.hex(), low)
    assert seen == {0, 2, 3, 4}


# ---- ptxas report ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kernel", ["secp256k1_ecrecover_kernel", "secp256k1_gtab_build"])
def test_ptxas_report_matches_design(kernel):
    log = os.path.join(CSRC, "build", "secp256k1.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("secp256k1.ptxas.log not built")
    m = re.search(r"Function properties for \w*" + kernel + r"\w*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads\nptxas info\s*: Used (\d+) registers", open(log).read())
    assert m, f"no ptxas report for {kernel}"
    stack, stores, loads, regs = map(int, m.groups())
    design = open(os.path.join(ROOT, "DESIGN.md")).read()
    row = re.search(r"^\| `" + kernel + r"` \| (\d+) \| (\d+) \| (\d+) \| (\d+) / (\d+) \|", design, re.M)
    assert row, f"DESIGN.md section 4.10 has no row for {kernel}"
    assert tuple(map(int, row.groups()[1:])) == (regs, stack, stores, loads)
