"""EIP-7594 cell recovery on the CPU: the consensus-specs route (tests/kzg_recover_ref.py) gets a blob's coefficients back
from every cell pattern the device tests use, and the device's per-column Lagrange route, with the kernel's indexing,
agrees with it coefficient for coefficient."""
import numpy as np
import pytest

import bls_ref as bls
import kzg_cells_ref as cells_ref
import kzg_recover_ref as ref
import kzg_ref

PATTERNS = ref.patterns(seed=7594)


def _blob(kind):
    if kind == "random":
        rng = np.random.default_rng(4844)
        return kzg_ref.to_blob([int.from_bytes(rng.bytes(32), "big") % bls.R for _ in range(4096)])
    return kzg_ref.to_blob([pow(w, kind, bls.R) for w in kzg_ref.roots_brp()])  # p = X^kind


@pytest.fixture(scope="module")
def random_blob():
    blob = _blob("random")
    return cells_ref.coefficients(blob), cells_ref.compute_cells(blob)


@pytest.mark.parametrize("name", sorted(PATTERNS))
def test_spec_route_recovers_the_blob(random_blob, name):
    coeffs, cells = random_blob
    idx = PATTERNS[name]
    assert ref.recover_coefficients(idx, [cells[c] for c in idx]) == coeffs


@pytest.mark.parametrize("name", ["first64", "last64", "odd", "random65", "shuffled"])
def test_column_route_agrees_with_spec_route(random_blob, name):
    coeffs, cells = random_blob
    idx = PATTERNS[name]
    given = [cells[c] for c in idx]
    assert ref.recover_columns(idx, given) == ref.recover_coefficients(idx, given) == coeffs


@pytest.mark.parametrize("e", [4095, 64, 63])
def test_monomials(e):
    blob = _blob(e)
    cells = cells_ref.compute_cells(blob)
    idx = PATTERNS["random64"]
    want = [0] * 4096
    want[e] = 1
    assert ref.recover_columns(idx, [cells[c] for c in idx]) == want


def test_column_route_reads_only_the_first_64_cells(random_blob):
    coeffs, cells = random_blob
    idx = PATTERNS["random96"]
    given = [cells[c] for c in idx]
    given[64] = bytes(2048)  # the 65th cell is not part of the interpolation: only the consistency check sees it
    assert ref.recover_columns(idx, given) == coeffs
