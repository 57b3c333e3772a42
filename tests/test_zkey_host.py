"""CPU checks of Groth16 from circom artifacts: the .zkey / .wtns oracle (tests/zkey_ref.py) against itself and the
verification equation, and a CPU build of the library's parser (ethrex_b200/csrc/zkey_parse.cpp with
tests/zkey_parse_check.cpp) fed valid files and every kind of malformed one, each refused with its status and a message
naming the section and field.  Finally the ptxas report of the new kernels against DESIGN.md section 4.16."""
import os
import re
import struct
import subprocess

import pytest

import zkey_ref as zr

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "ethrex_b200", "csrc")
OK, NOT_IN_FIELD, INVALID, UNSUPPORTED = 0, 2, 4, 8


@pytest.fixture(scope="module")
def circuit():
    return zr.ZkeyCircuit(n_constraints=11, n_public=2)


@pytest.fixture(scope="module")
def parser(tmp_path_factory):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    d = tmp_path_factory.mktemp("zkey")
    exe = str(d / "zkey_parse_check")
    subprocess.check_call([nvcc, "-std=c++17", "-O2", "-I", CSRC, "-o", exe, os.path.join(HERE, "zkey_parse_check.cpp"),
                           os.path.join(CSRC, "zkey_parse.cpp")])
    counter = [0]

    def run(items):
        """items: (kind, bytes[, n_vars]) -> [(status, message)]"""
        lines = []
        for it in items:
            counter[0] += 1
            path = str(d / f"f{counter[0]}")
            with open(path, "wb") as f:
                f.write(it[1])
            lines.append(f"{it[0]} {path}" + (f" {it[2]}" if len(it) > 2 else ""))
        out = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True, timeout=300).stdout.splitlines()
        assert len(out) == len(lines)
        return [(int(line.split(" ", 1)[0]), line.split(" ", 1)[1]) for line in out]
    return run


# ---- the oracle -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_constraints,n_public", [(5, 1), (11, 2), (20, 3), (27, 3)])
def test_oracle_h_two_ways_and_verification(n_constraints, n_public):
    c = zr.ZkeyCircuit(n_constraints, n_public, seed=n_constraints)
    assert c.n_constraints & (c.n_constraints - 1)  # not a power of two
    assert c.n >= c.n_constraints + n_public + 1
    z = c.assign([1234 + i for i in range(n_public)])
    a, b, cc = c.evaluations(z)
    assert all(x * y % zr.R == w for x, y, w in zip(a, b, cc))
    h1, h2 = c.h_terms(z)
    assert h1 == h2
    # the R1CS holds, so h(tau) Z(tau) is also (sum z u)(sum z v) - sum z w
    at = sum(x * y for x, y in zip(z, c.u)) % zr.R
    bt = sum(x * y for x, y in zip(z, c.v)) % zr.R
    ct = sum(x * y for x, y in zip(z, c.w)) % zr.R
    assert (at * bt - ct) % zr.R == h1
    for r, s in ((0, 0), (5, 9), (zr.R - 1, zr.R - 1)):
        assert c.verifies(z, r, s)
    # a different public input does not verify the same proof scalars
    a_, b_, c_ = c.proof_scalars(z, 3, 4)
    ic = sum(zz * c.k[i] for i, zz in enumerate([1] + [9] * n_public)) * pow(c.gamma, -1, zr.R) % zr.R
    assert (a_ * b_ - c.alpha * c.beta - c.gamma * ic - c.delta * c_) % zr.R != 0


def test_oracle_has_signals_outside_a_and_b(circuit):
    unused = [i for i in range(circuit.n_vars) if circuit.u[i] == 0 and circuit.v[i] == 0]
    assert len(unused) >= 3
    assert zr.g1_native(0) == bytes(64)


# ---- the parser -----------------------------------------------------------------------------------------------------------
def _zkey(sections, magic=b"zkey", version=1):
    return zr.container(magic, version, sections)


def _replace(sections, sid, payload):
    return [(i, payload if i == sid else p) for i, p in sections]


def test_parser_accepts_valid_files(circuit, parser):
    secs = circuit.sections()
    z = circuit.assign([3, 4])
    rev = list(reversed(secs))
    no10 = [s for s in secs if s[0] != 10]
    res = parser([("zkey", _zkey(secs)), ("zkey", _zkey(rev)), ("zkey", _zkey(no10)), ("zkey", _zkey(secs + [(11, b"x")])),
                  ("wtns", circuit.wtns(z), circuit.n_vars)])
    nrec = sum(len(r) for r in circuit.A) + sum(len(r) for r in circuit.B)
    for st, msg in res[:4]:
        assert (st, msg) == (OK, f"ok {circuit.n_vars} {circuit.n_public} {circuit.log_n} {nrec}")
    assert res[4] == (OK, "ok")


def test_parser_refuses_truncation_at_every_boundary(circuit, parser):
    data = _zkey(circuit.sections())
    cuts = [0, 4, 11]
    off = 12
    for sid, payload in circuit.sections():
        cuts += [off, off + 11, off + 12, off + 12 + len(payload) - 1]
        off += 12 + len(payload)
    cuts = sorted(set(c for c in cuts if c < len(data)))
    res = parser([("zkey", data[:c]) for c in cuts])
    for c, (st, msg) in zip(cuts, res):
        assert st == INVALID and "truncated" in msg, (c, msg)
    w = circuit.wtns(circuit.assign([3, 4]))
    res = parser([("wtns", w[:c], circuit.n_vars) for c in (0, 11, 12, 23, 24 + 39, len(w) - 1)])
    assert all(st == INVALID and "truncated" in msg for st, msg in res), res


def test_parser_refusals(circuit, parser):
    secs = circuit.sections()
    hdr = dict(secs)[2]
    nv, npub, n = circuit.n_vars, circuit.n_public, circuit.n

    def hdr_with(off, blob):
        return _replace(secs, 2, hdr[:off] + blob + hdr[off + len(blob):])

    recs = circuit.records()

    def with_record(rec, raw_value=None):
        body = zr.coef_record(*rec) if raw_value is None else struct.pack("<III", *rec[:3]) + raw_value
        payload = struct.pack("<I", len(recs) + 1) + b"".join(zr.coef_record(*r) for r in recs[:5]) + body + \
            b"".join(zr.coef_record(*r) for r in recs[5:])
        return _replace(secs, 4, payload)

    cases = [
        ("magic", _zkey(secs, magic=b"zkez"), INVALID, "magic"),
        ("version", _zkey(secs, version=2), UNSUPPORTED, "version 2"),
        ("plonk", _zkey(_replace(secs, 1, struct.pack("<I", 2))), UNSUPPORTED, "section 1: protocol 2"),
        ("foreign_q", _zkey(hdr_with(4, (zr.P - 2).to_bytes(32, "little"))), UNSUPPORTED, "section 2: q"),
        ("foreign_r", _zkey(hdr_with(40, (zr.R + 2).to_bytes(32, "little"))), UNSUPPORTED, "section 2: r"),
        ("n8q", _zkey(hdr_with(0, struct.pack("<I", 48))), UNSUPPORTED, "section 2: n8q = 48"),
        ("n8r", _zkey(hdr_with(36, struct.pack("<I", 48))), UNSUPPORTED, "section 2: n8r = 48"),
        ("domain_not_pow2", _zkey(hdr_with(80, struct.pack("<I", n + 1))), INVALID, "not a power of two"),
        ("domain_2_28", _zkey(hdr_with(80, struct.pack("<I", 1 << 28))), UNSUPPORTED, "2^28"),
        ("npublic_too_big", _zkey(hdr_with(76, struct.pack("<I", nv))), INVALID, "nPublic"),
        ("missing_5", _zkey([s for s in secs if s[0] != 5]), INVALID, "section 5 is missing"),
        ("duplicate_7", _zkey(secs + [(7, dict(secs)[7])]), INVALID, "section 7 appears twice"),
        ("trailing", _zkey(secs) + b"\0", INVALID, "trailing"),
        ("header_size", _zkey(_replace(secs, 2, hdr + b"\0" * 4)), INVALID, "section 2 (header)"),
        ("protocol_size", _zkey(_replace(secs, 1, b"\1\0\0\0\0")), INVALID, "section 1"),
        ("ic_count", _zkey(_replace(secs, 3, dict(secs)[3][:-64])), INVALID, "section 3 (IC)"),
        ("coef_count", _zkey(_replace(secs, 4, struct.pack("<I", len(recs) + 1) + dict(secs)[4][4:])), INVALID, "section 4 (coefficients)"),
        ("a_count", _zkey(_replace(secs, 5, dict(secs)[5] + bytes(64))), INVALID, "section 5 (A)"),
        ("b1_count", _zkey(_replace(secs, 6, dict(secs)[6][:-64])), INVALID, "section 6 (B1)"),
        ("b2_count", _zkey(_replace(secs, 7, dict(secs)[7][:-128])), INVALID, "section 7 (B2)"),
        ("c_count", _zkey(_replace(secs, 8, dict(secs)[8] + bytes(64))), INVALID, "section 8 (C)"),
        ("h_count", _zkey(_replace(secs, 9, dict(secs)[9][:-64])), INVALID, "section 9 (H)"),
        ("matrix_2", _zkey(with_record((2, 0, 1, 5))), INVALID, "record 5: matrix"),
        ("constraint_oob", _zkey(with_record((0, n, 1, 5))), INVALID, "record 5: constraint >= domainSize"),
        ("signal_oob", _zkey(with_record((1, 3, nv, 5))), INVALID, "record 5: signal >= nVars"),
        ("value_ge_r", _zkey(with_record((1, 3, 1, 0), zr.R.to_bytes(32, "little"))), NOT_IN_FIELD, "record 5: value >= r"),
    ]
    res = parser([("zkey", data) for _, data, _, _ in cases])
    for (name, _, st, frag), (got_st, msg) in zip(cases, res):
        assert got_st == st and frag in msg, (name, got_st, msg)
    # the edges that stay valid: the last constraint and signal, the largest value
    edge = parser([("zkey", _zkey(with_record((0, n - 1, nv - 1, 0), (zr.R - 1).to_bytes(32, "little"))))])
    assert edge[0][0] == OK, edge


def test_wtns_refusals(circuit, parser):
    z = circuit.assign([3, 4])
    nv = circuit.n_vars
    good = circuit.wtns(z)
    secs = [(1, struct.pack("<I", 32) + zr.R.to_bytes(32, "little") + struct.pack("<I", nv)), (2, b"".join(zr.le32(v) for v in z))]
    cases = [
        ("prime", zr.wtns_bytes(z, prime=zr.P), UNSUPPORTED, "prime"),
        ("n8", zr.wtns_bytes(z, prime=zr.R, n8=48), UNSUPPORTED, "n8 = 48"),
        ("count", zr.wtns_bytes(z + [7]), INVALID, f"nWitness {nv + 1}, the key has nVars {nv}"),
        ("values_size", zr.container(b"wtns", 2, [secs[0], (2, secs[1][1][:-32])]), INVALID, "section 2 (values)"),
        ("magic", b"wtnz" + good[4:], INVALID, "magic"),
        ("version", zr.container(b"wtns", 1, secs), UNSUPPORTED, "version 1"),
        ("missing", zr.container(b"wtns", 2, secs[:1]), INVALID, "section 2 is missing"),
        ("duplicate", zr.container(b"wtns", 2, secs + secs[1:]), INVALID, "section 2 appears twice"),
    ]
    res = parser([("wtns", data, nv) for _, data, _, _ in cases])
    for (name, _, st, frag), (got_st, msg) in zip(cases, res):
        assert got_st == st and frag in msg, (name, got_st, msg)
    # values >= r pass the parser: the device checks them
    assert parser([("wtns", zr.wtns_bytes([zr.R] * nv), nv)]) == [(OK, "ok")]


# ---- ptxas report ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kernel", ["zkey_eval", "zkey_eval_fixup", "zkey_coef_count", "zkey_coef_scatter", "zkey_wtns_check", "zkey_words_check"])
def test_ptxas_report_matches_design(kernel):
    log = os.path.join(CSRC, "build", "zkey.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("zkey.ptxas.log not built")
    m = re.search(r"Function properties for \w*\d" + kernel + r"E\w*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads\nptxas info\s*: Used (\d+) registers", open(log).read())
    assert m, f"no ptxas report for {kernel}"
    stack, stores, loads, regs = map(int, m.groups())
    design = open(os.path.join(ROOT, "DESIGN.md")).read()
    row = re.search(r"^\| `" + kernel + r"` \| (\d+) \| (\d+) \| (\d+) \| (\d+) / (\d+) \|", design, re.M)
    assert row, f"DESIGN.md section 4.16 has no row for {kernel}"
    assert tuple(map(int, row.groups()[1:])) == (regs, stack, stores, loads)
