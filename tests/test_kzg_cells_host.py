"""CPU checks of the EIP-7594 cell oracle (tests/kzg_cells_ref.py), independent of the device: the extension is systematic
and a Reed-Solomon codeword of p, and the universal verification equation holds for honest cell proofs over a known-tau
setup, as a scalar identity and through the pairing, and fails for a proof of the wrong cell.  Also the ptxas report of the
new kernels."""
import os
import re

import numpy as np
import pytest

import bls_ref as bls
import kzg_cells_ref as ref
import kzg_ref

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "ethrex_b200", "csrc")
R = bls.R
TAU = 0x2F1B7C93D4A5E6F708192A3B4C5D6E7F8091A2B3C4D5E6F708192A3B4C5D6E7F % R
CHALLENGE = 0x5A17C0FFEE0123456789ABCDEF0123456789ABCDEF0123456789ABCDEF01234 % R


def _blob(seed):
    rng = np.random.default_rng(seed)
    return kzg_ref.to_blob([int.from_bytes(rng.bytes(32), "big") % R for _ in range(4096)])


@pytest.fixture(scope="module")
def blob():
    return _blob(7594)


@pytest.fixture(scope="module")
def cells(blob):
    return ref.compute_cells(blob)


def test_first_half_is_the_blob(blob, cells):
    assert len(cells) == 128 and all(len(c) == 2048 for c in cells)
    assert b"".join(cells[:64]) == blob


def test_cells_are_one_polynomial_of_degree_below_4096(blob, cells):
    vals = [v for c in cells for v in ref.cell_values(c)]
    nat = [0] * 8192
    for i, v in enumerate(vals):
        nat[bls.bit_reverse(i, 13)] = v
    coeffs = ref.ntt(nat, pow(ref.ROOT_8192, -1, R))
    assert all(c == 0 for c in coeffs[4096:])
    # the second half against p evaluated through the Lagrange basis of the blob's own domain (no NTT involved)
    poly = kzg_ref.blob_values(blob)
    for k in (64, 65, 100, 127):
        xs = ref.coset(k)
        for t in (0, 13, 63):
            assert ref.cell_values(cells[k])[t] == kzg_ref.evaluate_direct(poly, xs[t])


def test_special_blobs():
    assert ref.compute_cells(bytes(131072)) == [bytes(2048)] * 128
    const = kzg_ref.to_blob([R - 1] * 4096)  # p = r - 1 everywhere: the extension is constant too
    assert ref.compute_cells(const) == [kzg_ref.to_blob([R - 1] * 64)] * 128


def test_coset_is_the_roots_of_x64_minus_shift():
    for k in (0, 1, 64, 127):
        s = ref.shift64(k)
        assert all(pow(x, 64, R) == s for x in ref.coset(k))
        assert len(set(ref.coset(k))) == 64
    assert len({ref.shift64(k) for k in range(128)}) == 128


def test_equation_holds_in_the_exponent(blob, cells):
    pt, qs = ref.proof_scalars(blob, TAU)
    assert ref.equation_in_exponent(TAU, CHALLENGE, [pt], cells, qs)
    assert ref.equation_in_exponent(TAU, 1, [pt], cells, qs)
    wrong = qs[:]
    wrong[6] = qs[5]  # the proof of cell 5 in cell 6's place
    assert not ref.equation_in_exponent(TAU, CHALLENGE, [pt], cells, wrong)
    bad_cells = cells[:]
    bad_cells[70] = (int.from_bytes(cells[70][:32], "big") ^ 1).to_bytes(32, "big") + cells[70][32:]
    assert not ref.equation_in_exponent(TAU, CHALLENGE, [pt], bad_cells, qs)


def test_equation_holds_through_the_pairing(blob, cells):
    commitments, proofs = ref.bundle([blob], TAU)
    assert commitments[0] == bls.compress(bls.mul(ref.horner(ref.coefficients(blob), TAU), bls.G1))
    assert ref.equation_by_pairing(TAU, CHALLENGE, commitments, cells, proofs)
    wrong = proofs[:]
    wrong[6] = proofs[5]
    assert not ref.equation_by_pairing(TAU, CHALLENGE, commitments, cells, wrong)


KERNELS = [("kzg_cells", k) for k in ("kzg_cells_tw_build", "kzg_cells_extend", "kzg_cells_weights", "kzg_cells_interp",
                                      "kzg_cells_interp_eval", "kzg_cells_scalars")] + [("bls_pairing", "kzg_cell_fold")]


def _ptxas(unit, kernel):
    log = os.path.join(CSRC, "build", unit + ".ptxas.log")
    if not os.path.exists(log):
        pytest.skip(f"{unit}.ptxas.log not built")
    m = re.search(r"Function properties for \w*\d" + kernel + r"E\w*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n"
                  r"ptxas info\s*: Used (\d+) registers", open(log).read())
    assert m, f"no ptxas report for {kernel}"
    return int(m.group(4)), int(m.group(1)), int(m.group(2)), int(m.group(3))


@pytest.mark.parametrize("unit,kernel", KERNELS)
def test_ptxas_rows_match_design(unit, kernel):
    """DESIGN.md lists each new kernel as | `kernel` | threads | registers | stack | spill stores / loads |; none spills"""
    regs, stack, st, ld = _ptxas(unit, kernel)
    assert st == 0 and ld == 0
    design = open(os.path.join(os.path.dirname(HERE), "DESIGN.md")).read()
    row = re.search(r"\| `" + kernel + r"` \| \d+ \| (\d+) \| (\d+) \| (\d+) / (\d+) \|", design)
    assert row, f"DESIGN.md has no ptxas row for {kernel}"
    assert tuple(int(g) for g in row.groups()) == (regs, stack, st, ld)
