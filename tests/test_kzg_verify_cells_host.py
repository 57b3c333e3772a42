"""CPU checks of verify_cell_kzg_proof_batch over arbitrary cells (b200zk_kzg_verify_cells): the spec-restating oracle
(tests/kzg_verify_cells_ref.py) in the exponent and through the pairing, its challenge against DESIGN section 4.12's for
whole blobs, the device's column route to A = sum r^k I_k, then a CPU build of the library's host unit
(ethrex_b200/csrc/cell_batch.cpp with tests/cell_batch_check.cpp) against the oracle's deduplication, commitment
indices, groupings and challenge byte for byte.  Finally the ptxas report of the new kernels against DESIGN.md 4.19."""
import os
import random
import re
import struct
import subprocess

import numpy as np
import pytest

import bls_ref as bls
import kzg_cells_ref as cref
import kzg_ref
import kzg_verify_cells_ref as ref

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "ethrex_b200", "csrc")
R = bls.R
TAU = 0x2F1B7C93D4A5E6F708192A3B4C5D6E7F8091A2B3C4D5E6F708192A3B4C5D6E7F % R
CHALLENGE = 0x5A17C0FFEE0123456789ABCDEF0123456789ABCDEF0123456789ABCDEF01234 % R


def _blob(seed):
    rng = np.random.default_rng(seed)
    return kzg_ref.to_blob([int.from_bytes(rng.bytes(32), "big") % R for _ in range(4096)])


@pytest.fixture(scope="module")
def scalars():
    """two blobs: their cells, and the logs of their commitments and 128 proofs each"""
    out = []
    for seed in (11, 12):
        blob = _blob(seed)
        pt, qs = cref.proof_scalars(blob, TAU)
        out.append((cref.compute_cells(blob), pt, qs))
    return out


@pytest.fixture(scope="module")
def points():
    """one blob with its points: (cells, commitment, 128 proofs)"""
    blob = _blob(13)
    cs, ps = cref.bundle([blob], TAU)
    return cref.compute_cells(blob), cs[0], ps


def _pick(scalars, pairs):
    """(commitment logs, cell indices, cells, proof logs) of the (blob, cell) pairs"""
    return ([scalars[b][1] for b, _ in pairs], [c for _, c in pairs], [scalars[b][0][c] for b, c in pairs],
            [scalars[b][2][c] for b, c in pairs])


def test_honest_subsets_hold_in_the_exponent(scalars):
    rng = random.Random(1)
    subsets = [
        [(b, 5) for b in (0, 1)],                                      # one column
        [(b, c) for b in (0, 1) for c in rng.sample(range(128), 8)],  # 8 random columns
        [(0, c) for c in rng.sample(range(128), 64)],                  # half a blob
        [(1, 3)],                                                      # one cell
        [(0, 7), (1, 7), (0, 7), (1, 100), (0, 7)],                   # repeated cells, shared commitments
        rng.sample([(b, c) for b in (0, 1) for c in range(128)], 256),  # everything, shuffled
    ]
    for pairs in subsets:
        assert ref.equation_in_exponent(TAU, CHALLENGE, *_pick(scalars, pairs))
        assert ref.equation_in_exponent(TAU, 1, *_pick(scalars, pairs))


def test_tampered_subsets_fail_in_the_exponent(scalars):
    pairs = [(0, 3), (1, 3), (0, 90), (1, 17), (0, 64)]
    p, idx, cells, q = _pick(scalars, pairs)
    assert ref.equation_in_exponent(TAU, CHALLENGE, p, idx, cells, q)
    swapped = q[:]
    swapped[2], swapped[3] = q[3], q[2]
    assert not ref.equation_in_exponent(TAU, CHALLENGE, p, idx, cells, swapped)
    moved = q[:]
    moved[1] = q[0]  # blob 0's proof of cell 3 for blob 1's cell 3
    assert not ref.equation_in_exponent(TAU, CHALLENGE, p, idx, cells, moved)
    assert not ref.equation_in_exponent(TAU, CHALLENGE, p, [4] + idx[1:], cells, q)
    changed = cells[:]
    v = (cref.cell_values(cells[4])[9] + 1) % R
    changed[4] = cells[4][:32 * 9] + v.to_bytes(32, "big") + cells[4][32 * 10:]
    assert not ref.equation_in_exponent(TAU, CHALLENGE, p, idx, changed, q)
    assert not ref.equation_in_exponent(TAU, CHALLENGE, [p[1], p[0]] + p[2:], idx, cells, q)


def test_column_route_is_the_sum_of_interpolants(scalars):
    rng = random.Random(2)
    pairs = [(b, c) for b in (0, 1) for c in rng.sample(range(128), 6)] + [(0, 0), (0, 0), (1, 127)]
    _, idx, cells, _ = _pick(scalars, pairs)
    want = sum(pow(CHALLENGE, k, R) * cref.interpolate_at(c, cref.cell_values(y), TAU) for k, (c, y) in enumerate(zip(idx, cells))) % R
    assert cref.horner(ref.column_route(CHALLENGE, idx, cells), TAU) == want
    # a column's interpolant of the blob's own cell is p mod (X^64 - s_c)
    blob_coeffs = cref.coefficients(b"".join(scalars[0][0][:64]))
    s = cref.shift64(77)
    folded = [sum(blob_coeffs[64 * m + j] * pow(s, m, R) for m in range(64)) % R for j in range(64)]
    assert ref.column_route(1, [77], [scalars[0][0][77]]) == folded


def test_pairing_accepts_honest_and_rejects_tampered(points):
    cells, cm, ps = points
    idx = [9, 100, 9, 33]
    args = ([cm] * 4, idx, [cells[c] for c in idx], [ps[c] for c in idx])
    assert ref.verify(TAU, *args)
    wrong = list(args[3])
    wrong[1], wrong[3] = wrong[3], wrong[1]
    assert not ref.verify(TAU, args[0], idx, args[2], wrong)
    assert ref.verify(TAU, [], [], [], [])


def test_challenge_is_section_4_12_for_whole_blobs():
    rng = random.Random(3)
    cms = [rng.randbytes(48) for _ in range(3)]
    cells = [rng.randbytes(2048) for _ in range(3 * 128)]
    proofs = [rng.randbytes(48) for _ in range(3 * 128)]
    per_cell = [cms[k // 128] for k in range(3 * 128)]
    idx = [k % 128 for k in range(3 * 128)]
    assert ref.challenge(per_cell, idx, cells, proofs) == ref.whole_blob_challenge(cms, cells, proofs)
    # a repeated commitment is listed once: the constructions part
    dup = [cms[0], cms[0], cms[2]]
    per_cell = [dup[k // 128] for k in range(3 * 128)]
    assert ref.challenge(per_cell, idx, cells, proofs) != ref.whole_blob_challenge(dup, cells, proofs)


# ---- the host unit --------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def host(tmp_path_factory):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    d = tmp_path_factory.mktemp("cell_batch")
    exe = str(d / "cell_batch_check")
    subprocess.check_call([nvcc, "-std=c++17", "-O2", "-I", CSRC, "-o", exe, os.path.join(HERE, "cell_batch_check.cpp"),
                           os.path.join(CSRC, "cell_batch.cpp")])
    counter = [0]

    def run(cases):
        """cases: (commitments, indices, cells, proofs) -> one answer line each"""
        paths = []
        for cm, idx, cells, proofs in cases:
            counter[0] += 1
            path = str(d / f"c{counter[0]}")
            with open(path, "wb") as f:
                f.write(struct.pack("<Q", len(idx)) + b"".join(cm) + struct.pack(f"<{len(idx)}Q", *idx) + b"".join(cells) + b"".join(proofs))
            paths.append(path)
        out = subprocess.run([exe], input="\n".join(paths) + "\n", capture_output=True, text=True, check=True, timeout=300).stdout.splitlines()
        assert len(out) == len(cases)
        return out
    return run


def _expected(cm, idx, cells, proofs):
    unique, index = ref.deduplicate(cm)
    first = [cm.index(u) for u in unique]

    def csr(keys, order):
        off, by = [0], []
        for key in order:
            members = [k for k, x in enumerate(keys) if x == key]
            by += members
            off.append(len(by))
        return off, by
    commit_off, by_commit = csr(index, range(len(unique)))
    columns = sorted(set(idx))
    column_off, by_column = csr(idx, columns)
    j = lambda v: ",".join(str(x) for x in v)  # noqa: E731
    r = ref.challenge(cm, idx, cells, proofs)
    return (f"ok unique={j(first)} index={j(index)} commit_off={j(commit_off)} by_commit={j(by_commit)} columns={j(columns)} "
            f"column_off={j(column_off)} by_column={j(by_column)} r={r:064x}")


def _case(rng, n, n_commit, n_index=128, repeat=0):
    pool = [rng.randbytes(48) for _ in range(n_commit)]
    cm = [rng.choice(pool) for _ in range(n)]
    idx = [rng.randrange(n_index) for _ in range(n)]
    cells = [rng.randbytes(2048) for _ in range(n)]
    proofs = [rng.randbytes(48) for _ in range(n)]
    for _ in range(repeat):  # whole cells repeated
        a, b = rng.randrange(n), rng.randrange(n)
        cm[b], idx[b], cells[b], proofs[b] = cm[a], idx[a], cells[a], proofs[a]
    return cm, idx, cells, proofs


def test_host_unit_matches_the_oracle(host):
    rng = random.Random(4)
    cases = [_case(rng, 40, 40), _case(rng, 300, 300), _case(rng, 200, 5, repeat=30), _case(rng, 64, 1, n_index=3, repeat=10),
             _case(rng, 1, 1), _case(rng, 0, 1), _case(rng, 128 * 3, 3)]
    # whole blobs, shuffled
    cm, idx, cells, proofs = _case(rng, 256, 2)
    order = list(range(256))
    rng.shuffle(order)
    cases.append(([cm[k] for k in order], [k % 128 for k in order], [cells[k] for k in order], [proofs[k] for k in order]))
    assert host(cases) == [_expected(*c) for c in cases]


def test_host_unit_refuses_indices_from_128(host):
    rng = random.Random(5)
    cm, idx, cells, proofs = _case(rng, 10, 3)
    cases = []
    for pos, bad in ((0, 128), (7, 2 ** 64 - 1), (9, 200)):
        i = idx[:]
        i[pos] = bad
        cases.append((cm, i, cells, proofs))
    two = idx[:]
    two[4], two[6] = 129, 128
    cases.append((cm, two, cells, proofs))
    assert host(cases) == ["bad 0", "bad 7", "bad 9", "bad 4"]


def test_host_challenge_matches_whole_blob_construction(host):
    rng = random.Random(6)
    cms = [rng.randbytes(48) for _ in range(2)]
    cells = [rng.randbytes(2048) for _ in range(256)]
    proofs = [rng.randbytes(48) for _ in range(256)]
    line = host([([cms[k // 128] for k in range(256)], [k % 128 for k in range(256)], cells, proofs)])[0]
    assert line.endswith(f"r={ref.whole_blob_challenge(cms, cells, proofs):064x}")


KERNELS = ["kzg_vcells_powers", "kzg_vcells_weights", "kzg_vcells_columns"]


def _ptxas(kernel):
    log = os.path.join(CSRC, "build", "kzg_cells.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("kzg_cells.ptxas.log not built")
    m = re.search(r"Function properties for \w*\d" + kernel + r"E\w*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n"
                  r"ptxas info\s*: Used (\d+) registers", open(log).read())
    assert m, f"no ptxas report for {kernel}"
    return int(m.group(4)), int(m.group(1)), int(m.group(2)), int(m.group(3))


@pytest.mark.parametrize("kernel", KERNELS)
def test_ptxas_rows_match_design(kernel):
    """DESIGN.md 4.19 lists each new kernel as | `kernel` | threads | registers | stack | spill stores / loads |; none spills"""
    regs, stack, st, ld = _ptxas(kernel)
    assert st == 0 and ld == 0
    design = open(os.path.join(ROOT, "DESIGN.md")).read()
    row = re.search(r"\| `" + kernel + r"` \| \d+ \| (\d+) \| (\d+) \| (\d+) / (\d+) \|", design)
    assert row, f"DESIGN.md has no ptxas row for {kernel}"
    assert tuple(int(g) for g in row.groups()) == (regs, stack, st, ld)
