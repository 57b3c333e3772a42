"""CPU checks of PLONK from circom artifacts: the snarkjs 0.7 oracle (tests/plonk_ref.py) against its own verifier and the
pairing, T by snarkjs's root-domain route against the device's coset route, and a CPU build of the library's PLONK key
parser (plonk_zkey_parse in ethrex_b200/csrc/zkey_parse.cpp, with tests/plonk_parse_check.cpp) fed valid keys and every
kind of malformed one, each refused with its status and a message naming the section and field."""
import os
import struct
import subprocess

import pytest

import plonk_ref as pr
from zkey_ref import container

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "ethrex_b200", "csrc")
OK, NOT_IN_FIELD, INVALID, UNSUPPORTED = 0, 2, 4, 8
R, P = pr.R, pr.P


@pytest.fixture(scope="module")
def circuit():
    return pr.PlonkCircuit(n_gates=9, n_public=2, n_private=3, n_additions=6, seed=7)


@pytest.fixture(scope="module")
def sections(circuit):
    return circuit.sections()


@pytest.fixture(scope="module")
def parser(tmp_path_factory):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    d = tmp_path_factory.mktemp("plonk")
    exe = str(d / "plonk_parse_check")
    subprocess.check_call([nvcc, "-std=c++17", "-O2", "-I", CSRC, "-o", exe, os.path.join(HERE, "plonk_parse_check.cpp"), os.path.join(CSRC, "zkey_parse.cpp")])
    counter = [0]

    def run(files):
        paths = []
        for data in files:
            counter[0] += 1
            paths.append(str(d / f"k{counter[0]}"))
            with open(paths[-1], "wb") as f:
                f.write(data)
        out = subprocess.run([exe], input="\n".join(paths) + "\n", capture_output=True, text=True, check=True, timeout=300).stdout.splitlines()
        assert len(out) == len(paths)
        return [(int(line.split(" ", 1)[0]), line.split(" ", 1)[1]) for line in out]
    return run


def zkey(sections):
    return container(b"zkey", 1, sections)


def patch(payload: bytes, off: int, data: bytes) -> bytes:
    return payload[:off] + data + payload[off + len(data):]


# ---- the oracle -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_gates,n_public,n_additions", [(9, 2, 6), (5, 0, 3), (20, 4, 9), (11, 1, 0)])
def test_oracle_t_two_routes_and_verification(n_gates, n_public, n_additions):
    c = pr.PlonkCircuit(n_gates=n_gates, n_public=n_public, n_additions=n_additions, seed=n_gates)
    assert c.n_constraints & (c.n_constraints - 1)  # not a power of two
    assert any(s1 >= c.n_wtns for s1, _, _, _ in c.adds) or n_additions < 2  # a chain of additions
    wt = c.assign([100 + i for i in range(n_public)])
    pub = c.public(wt)
    for blinding in ([0] * 11, [pr.R - 1] * 11, list(range(3, 14))):
        proof, info = c.prove(wt, blinding, route="root")
        proof2, info2 = c.prove(wt, blinding, route="coset")
        assert info["T"] == info2["T"] and proof == proof2
        assert c.verify(proof, pub, tau=c.tau)


def test_oracle_proof_passes_the_pairing_and_tampering_fails(circuit):
    wt = circuit.assign([5, 9])
    pub = circuit.public(wt)
    proof, _ = circuit.prove(wt, list(range(20, 31)))
    assert circuit.verify(proof, pub)  # the Python pairing
    for w in range(9):  # each commitment replaced by another curve point
        bad = proof[:64 * w] + pr._g1(1234 + w) + proof[64 * w + 64:]
        assert not circuit.verify(bad, pub, tau=circuit.tau), w
    for k in range(6):  # each evaluation
        off = 576 + 32 * k
        v = (int.from_bytes(proof[off:off + 32], "big") + 1) % R
        assert not circuit.verify(proof[:off] + v.to_bytes(32, "big") + proof[off + 32:], pub, tau=circuit.tau), k
    for i in range(len(pub)):
        assert not circuit.verify(proof, pub[:i] + [(pub[i] + 1) % R] + pub[i + 1:], tau=circuit.tau)


def test_oracle_refuses_unsatisfying_witnesses(circuit):
    wt = circuit.assign([5, 9])
    gate_out = 1 + circuit.n_public + 3  # the first gate's output
    broken = list(wt)
    broken[gate_out] = (broken[gate_out] + 1) % R
    with pytest.raises(ValueError, match="gates|copy"):
        circuit.prove(broken)


# ---- the parser -----------------------------------------------------------------------------------------------------------
def test_parser_accepts_the_oracle_keys(parser, circuit, sections):
    c0 = pr.PlonkCircuit(n_gates=5, n_public=0, n_additions=0, seed=3)
    got = parser([zkey(sections), zkey(list(reversed(sections))), c0.zkey()])
    want = f"ok {circuit.n_vars} {circuit.n_public} {circuit.log_n} {circuit.n_additions} {circuit.n_constraints}"
    assert got[0] == (OK, want) and got[1] == (OK, want)
    assert got[2][0] == OK


def test_parser_refuses_every_truncation(parser, sections):
    full = zkey(sections)
    cuts, off = [], 12
    for _, payload in sections:
        cuts += [off, off + 6, off + 12, off + 12 + len(payload) // 2]
        off += 12 + len(payload)
    res = parser([full[:c] for c in sorted(set(cuts)) if c < len(full)] + [full[:5], full + b"x"])
    for status, msg in res:
        assert status == INVALID and ("truncated" in msg or "trailing" in msg or "missing" in msg or "holds" in msg), msg


def test_parser_refuses_malformed_sections(parser, sections):
    s = dict(sections)
    h = s[2]
    cases = [
        (zkey(sections), OK, "ok"),
        (zkey([x for x in sections if x[0] != 12]), INVALID, "section 12 is missing"),
        (zkey(sections + [(5, s[5])]), INVALID, "appears twice"),
        (zkey(sections).replace(b"zkey", b"zkez", 1), INVALID, "magic"),
        (zkey([(1, struct.pack("<I", 1))] + sections[1:]), UNSUPPORTED, "protocol 1 is not PLONK"),
        (zkey([(1, struct.pack("<I", 10))] + sections[1:]), UNSUPPORTED, "protocol 10"),
        (zkey([(1, b"\x02\0\0")] + sections[1:]), INVALID, "section 1"),
        (zkey([sections[0], (2, patch(h, 0, struct.pack("<I", 48)))] + sections[2:]), UNSUPPORTED, "n8q = 48"),
        (zkey([sections[0], (2, patch(h, 4, (P + 2).to_bytes(32, "little")))] + sections[2:]), UNSUPPORTED, "q is not"),
        (zkey([sections[0], (2, patch(h, 36, struct.pack("<I", 48)))] + sections[2:]), UNSUPPORTED, "n8r = 48"),
        (zkey([sections[0], (2, patch(h, 40, (R + 2).to_bytes(32, "little")))] + sections[2:]), UNSUPPORTED, "r is not"),
        (zkey([sections[0], (2, h[:-1])] + sections[2:]), INVALID, "section 2 (header) holds 795"),
        (zkey([sections[0], (2, patch(h, 80, struct.pack("<I", 24)))] + sections[2:]), INVALID, "not a power of two"),
        (zkey([sections[0], (2, patch(h, 80, struct.pack("<I", 1 << 27)))] + sections[2:]), UNSUPPORTED, "2^27"),
        (zkey([sections[0], (2, patch(h, 80, struct.pack("<I", 4)))] + sections[2:]), UNSUPPORTED, "below 8"),
        (zkey([sections[0], (2, patch(h, 76, struct.pack("<I", 99)))] + sections[2:]), INVALID, "nPublic 99 exceeds nConstraints"),
        (zkey([sections[0], (2, patch(h, 88, struct.pack("<I", 999)))] + sections[2:]), INVALID, "nConstraints 999 exceeds domainSize"),
        (zkey([sections[0], (2, patch(h, 84, struct.pack("<I", 10 ** 6)))] + sections[2:]), INVALID, "nAdditions"),
        (zkey([sections[0], (2, patch(h, 72, struct.pack("<I", 1)))] + sections[2:]), INVALID, "nVars 1"),
        (zkey([sections[0], (2, patch(h, 92, R.to_bytes(32, "little")))] + sections[2:]), NOT_IN_FIELD, "k1 is >= r"),
        (zkey([sections[0], (2, patch(h, 124, (R + 5).to_bytes(32, "little")))] + sections[2:]), NOT_IN_FIELD, "k2 is >= r"),
        (zkey([sections[0], (2, patch(h, 156 + 64 * 3, P.to_bytes(32, "little")))] + sections[2:]), NOT_IN_FIELD, "Qo has a coordinate >= q"),
        (zkey([sections[0], (2, patch(h, 156 + 512 + 96, (P + 1).to_bytes(32, "little")))] + sections[2:]), NOT_IN_FIELD, "X_2 has a coordinate"),
    ]
    res = parser([c[0] for c in cases])
    for (_, status, frag), (got, msg) in zip(cases, res):
        assert got == status and frag in msg, (status, frag, got, msg)


def test_parser_refuses_bad_records_and_values(parser, circuit, sections):
    s = dict(sections)
    nw = circuit.n_wtns

    def with_section(sid, payload):
        return container(b"zkey", 1, [(k, payload if k == sid else v) for k, v in sections])
    bad_r = R.to_bytes(32, "little")
    cases = [
        (with_section(4, patch(s[4], 4 * 3, struct.pack("<I", circuit.n_vars))), INVALID, "section 4 (A map): entry 3 is signal"),
        (with_section(6, patch(s[6], 0, struct.pack("<I", circuit.n_vars + 7))), INVALID, "section 6 (C map): entry 0"),
        (with_section(3, patch(s[3], 72 * 2, struct.pack("<I", nw + 2))), INVALID, "addition 2 reads signal"),
        (with_section(3, patch(s[3], 72 * 0 + 4, struct.pack("<I", nw))), INVALID, "addition 0 reads signal"),
        (with_section(3, patch(s[3], 72 * 1 + 8, bad_r)), NOT_IN_FIELD, "addition 1: a factor"),
        (with_section(3, patch(s[3], 72 * 4 + 40, bad_r)), NOT_IN_FIELD, "addition 4: a factor"),
        (with_section(7, patch(s[7], 32 * 5, bad_r)), NOT_IN_FIELD, "section 7 (Qm): value 5"),
        (with_section(11, patch(s[11], 32 * (circuit.n + 3), bad_r)), NOT_IN_FIELD, "section 11 (Qc): value"),
        (with_section(12, patch(s[12], 32 * 11 * circuit.n, bad_r)), NOT_IN_FIELD, "section 12 (sigma)"),
        (with_section(13, patch(s[13], 32 * 6 * circuit.n, bad_r)), NOT_IN_FIELD, "section 13 (Lagrange)"),
        (with_section(14, patch(s[14], 64 * 3 + 32, P.to_bytes(32, "little"))), NOT_IN_FIELD, "section 14 (PTau): point 3"),
    ]
    for k in range(3, 15):
        cases.append((with_section(k, s[k] + bytes(4)), INVALID, f"section {k} ("))
    res = parser([c[0] for c in cases])
    for (_, status, frag), (got, msg) in zip(cases, res):
        assert got == status and frag in msg, (status, frag, got, msg)
