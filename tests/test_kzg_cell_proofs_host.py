"""CPU checks of EIP-7594 cell proofs by FK20, independent of the device: the proof of cell k expands to
pi_k = sum_(m=1..63) s_k^(m-1) T_m, and the FK20 bookkeeping of the kernels (tests/fk20_ref.py: table, column DFTs,
pointwise sums, inverse DFT, truncation, final DFT, bit reversal) reproduces every T_m and every proof, all in scalars over
a known tau.  Also the ptxas report of the new kernels."""
import os
import re

import numpy as np
import pytest

import bls_ref as bls
import fk20_ref as fk
import kzg_cells_ref as ref
import kzg_ref

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "ethrex_b200", "csrc")
R = bls.R
TAU = 0x2F1B7C93D4A5E6F708192A3B4C5D6E7F8091A2B3C4D5E6F708192A3B4C5D6E7F % R


def _blob(seed):
    rng = np.random.default_rng(seed)
    return kzg_ref.to_blob([int.from_bytes(rng.bytes(32), "big") % R for _ in range(4096)])


def _monomial_blob(e):
    return kzg_ref.to_blob([pow(w, e, R) for w in kzg_ref.roots_brp()])


BLOBS = [_blob(1), _blob(2), _monomial_blob(4095), _monomial_blob(64), _monomial_blob(63)]


@pytest.mark.parametrize("i", range(len(BLOBS)))
def test_identity_in_scalars(i):
    blob = BLOBS[i]
    assert fk.proofs_from_toeplitz(fk.toeplitz_direct(blob, TAU)) == ref.proof_scalars(blob, TAU)[1]


@pytest.mark.parametrize("i", range(len(BLOBS)))
def test_fk20_restated_reproduces_toeplitz_sums_and_proofs(i):
    blob = BLOBS[i]
    z = fk.toeplitz_sums(blob, TAU)
    assert z[1:64] == fk.toeplitz_direct(blob, TAU)[1:64]
    assert fk.proof_scalars(blob, TAU) == ref.proof_scalars(blob, TAU)[1]


def test_monomial_edges():
    # p = X^4095 runs the longest Toeplitz row: T_1 = tau^4031; p = X^63 has degree < 64, so every proof is 0
    assert fk.toeplitz_direct(BLOBS[2], TAU)[1] == pow(TAU, 4095 - 64, R)
    assert fk.proof_scalars(BLOBS[4], TAU) == [0] * 128
    t = fk.toeplitz_direct(BLOBS[3], TAU)  # p = X^64: T_1 = 1, the rest 0, so every proof is [1]1
    assert t[1] == 1 and not any(t[2:])
    assert fk.proof_scalars(BLOBS[3], TAU) == [1] * 128


def test_constant_blob_has_zero_proofs():
    assert fk.proof_scalars(kzg_ref.to_blob([R - 1] * 4096), TAU) == [0] * 128


KERNELS = ["kzg_fk20_table", "kzg_fk20_columns", "kzg_fk20_msm", "kzg_fk20_proofs"]


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
    """DESIGN.md lists each new kernel as | `kernel` | threads | registers | stack | spill stores / loads |; none spills"""
    regs, stack, st, ld = _ptxas(kernel)
    assert st == 0 and ld == 0
    design = open(os.path.join(os.path.dirname(HERE), "DESIGN.md")).read()
    row = re.search(r"\| `" + kernel + r"` \| \d+ \| (\d+) \| (\d+) \| (\d+) / (\d+) \|", design)
    assert row, f"DESIGN.md has no ptxas row for {kernel}"
    assert tuple(int(g) for g in row.groups()) == (regs, stack, st, ld)
