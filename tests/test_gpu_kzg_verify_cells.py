"""EIP-7594 cell-proof verification over arbitrary cells on the device (b200zk_kzg_verify_cells) over the synthetic
known-tau setup of tests/test_gpu_kzg_cells.py.  Cells and proofs come from the existing device calls (held against the
oracle of tests/kzg_cells_ref.py for the first blob).  Honest sets of cells in every shape verify, every tampered set
does not, each input rule gets its status and names the cell, and the answer agrees with the whole-blob call, with
KzgSettings, with the spec-restating oracle of tests/kzg_verify_cells_ref.py, and with recovery's output."""
import ctypes
import random

import numpy as np
import pytest

import bls_pairing_ref as B
import bls_ref as bls
import kzg_cells_ref as cref
import kzg_ref
import kzg_verify_cells_ref as ref

pytestmark = pytest.mark.gpu

import ethrex_b200 as eb  # noqa: E402
from ethrex_b200 import _ffi  # noqa: E402
from ethrex_b200.kzg import KzgSettings  # noqa: E402

TAU = 0x2F1B7C93D4A5E6F708192A3B4C5D6E7F8091A2B3C4D5E6F708192A3B4C5D6E7F % bls.R
IDENTITY = bytes([0xC0]) + bytes(47)
ZERO = 3  # the zero blob's place in the bundle
N_BLOBS = 24


@pytest.fixture(scope="module")
def points():
    return b"".join(bls.compress(p) for p in bls.generator_multiples(bls.lagrange_setup_scalars(TAU)))


@pytest.fixture(scope="module")
def monomial():
    return b"".join(bls.compress(p) for p in bls.generator_multiples([pow(TAU, i, bls.R) for i in range(4096)]))


@pytest.fixture(scope="module")
def g2_points():
    return cref.g2_setup(TAU)


@pytest.fixture(scope="module")
def setups(ctx, points, monomial, g2_points):
    g1 = ctx.bls12_381_g1_bases_upload(points, 4096)
    ctx.bases_precompute(g1, 0)
    g2 = ctx.bls12_381_g2_bases_upload(g2_points, 65)
    mono = ctx.bls12_381_g1_bases_upload(monomial, 4096)
    yield g1, g2, mono
    for h in (g1, g2, mono):
        ctx.bases_free(h)


@pytest.fixture(scope="module")
def bundle(ctx, setups):
    """24 blobs (the zero blob at 3): (blobs, commitments, cells[b][c], proofs[b][c]) from the device's cell and FK20 calls"""
    rng = np.random.default_rng(7594)
    blobs = [kzg_ref.to_blob([int.from_bytes(rng.bytes(32), "big") % bls.R for _ in range(4096)]) for _ in range(N_BLOBS)]
    blobs[ZERO] = bytes(131072)
    cells = ctx.kzg_compute_cells(b"".join(blobs))
    cs, ps = ctx.kzg_blob_to_commitment_and_cell_proofs(setups[0], setups[2], b"".join(blobs))
    proofs = [ps[128 * b:128 * (b + 1)] for b in range(N_BLOBS)]
    ocs, ops = cref.bundle(blobs[:1], TAU)
    assert (cs[0], proofs[0], cells[0]) == (ocs[0], ops, cref.compute_cells(blobs[0]))
    assert cs[ZERO] == IDENTITY and proofs[ZERO] == [IDENTITY] * 128
    return blobs, cs, cells, proofs


def _items(bundle, pairs):
    """(commitments, indices, cells, proofs) of the (blob, cell) pairs"""
    _, cs, cells, proofs = bundle
    return [cs[b] for b, _ in pairs], [c for _, c in pairs], [cells[b][c] for b, c in pairs], [proofs[b][c] for b, c in pairs]


def _verify(ctx, setups, cm, idx, cells, proofs):
    return ctx.kzg_verify_cells(setups[0], setups[1], cm, idx, cells, proofs)


def _honest_cases():
    rng = random.Random(7594)
    half = [(b, c) for b in range(6) for c in rng.sample(range(128), 64)]
    shuffled = [(b, c) for b in (1, 2) for c in range(128)]
    rng.shuffle(shuffled)
    cols = rng.sample(range(128), 8)
    return {
        "one_column_24_blobs": [(b, 37) for b in range(N_BLOBS)],
        "8_random_columns": [(b, c) for b in range(6) for c in cols],
        "half_of_each_blob": half,
        "all_128_shuffled": shuffled,
        "blob_twice": [(4, c) for c in range(0, 128, 3)] + [(5, 9)] + [(4, c) for c in range(1, 128, 5)],
        "repeated_cell": [(6, 11), (7, 20), (6, 11), (6, 11), (7, 21)],
        "zero_blob": [(ZERO, c) for c in range(0, 128, 7)],
        "zero_blob_and_others": [(ZERO, 5), (8, 5), (ZERO, 90), (9, 1)],
        "one_cell": [(10, 127)],
    }


@pytest.mark.parametrize("name", sorted(_honest_cases()))
def test_honest_cells_verify(ctx, setups, bundle, name):
    assert _verify(ctx, setups, *_items(bundle, _honest_cases()[name])) is True


def test_tampered_cells_fail(ctx, setups, bundle):
    pairs = [(b, c) for b in range(4) for c in (2, 40, 77, 120)]
    cm, idx, cells, proofs = _items(bundle, pairs)
    assert _verify(ctx, setups, cm, idx, cells, proofs) is True
    cases = []
    swapped = proofs[:]  # two proofs swapped
    swapped[1], swapped[6] = proofs[6], proofs[1]
    cases.append((cm, idx, cells, swapped))
    moved = proofs[:]  # blob 2's proof of cell 40 where blob 1's is due
    moved[5] = bundle[3][2][40]
    cases.append((cm, idx, cells, moved))
    reindexed = idx[:]  # one cell index changed to another
    reindexed[9] = 41
    cases.append((cm, reindexed, cells, proofs))
    changed = cells[:]  # one element of a cell changed
    v = (int.from_bytes(cells[11][32 * 9:32 * 10], "big") + 1) % bls.R
    changed[11] = cells[11][:32 * 9] + v.to_bytes(32, "big") + cells[11][32 * 10:]
    cases.append((cm, idx, changed, proofs))
    cswap = cm[:]  # commitments swapped between two cells
    cswap[0], cswap[4] = cm[4], cm[0]
    cases.append((cswap, idx, cells, proofs))
    ident = proofs[:]  # a proof replaced by the identity (on blob 0: the zero blob's proofs are the identity already)
    ident[1] = IDENTITY
    cases.append((cm, idx, cells, ident))
    assert [_verify(ctx, setups, *c) for c in cases] == [False] * len(cases)


def test_agrees_with_the_oracle(ctx, setups, bundle):
    pairs = [(0, 9), (0, 100), (1, 9), (0, 9)]
    items = _items(bundle, pairs)
    assert _verify(ctx, setups, *items) is ref.verify(TAU, *items) is True
    wrong = list(items[3])
    wrong[1], wrong[3] = wrong[3], wrong[1]
    assert _verify(ctx, setups, items[0], items[1], items[2], wrong) is ref.verify(TAU, items[0], items[1], items[2], wrong) is False


def test_agrees_with_the_whole_blob_call(ctx, setups, bundle):
    blobs, cs, cells, proofs = bundle
    for blob_ids in ((0,), (1, 2, 3, 4, 5, 6)):
        pairs = [(b, c) for b in blob_ids for c in range(128)]
        items = _items(bundle, pairs)
        whole = ctx.kzg_verify_cell_proof_batch(setups[0], setups[1], b"".join(blobs[b] for b in blob_ids), b"".join(cs[b] for b in blob_ids),
                                                b"".join(b"".join(proofs[b]) for b in blob_ids))
        assert _verify(ctx, setups, *items) is whole is True
        wrong = list(items[3])
        wrong[3] = items[3][4]
        whole = ctx.kzg_verify_cell_proof_batch(setups[0], setups[1], b"".join(blobs[b] for b in blob_ids), b"".join(cs[b] for b in blob_ids),
                                                b"".join(wrong))
        assert _verify(ctx, setups, items[0], items[1], items[2], wrong) is whole is False


def test_statuses(ctx, setups, bundle, g2_points):
    pairs = [(0, 1), (1, 2), (0, 3), (2, 4), (1, 5), (0, 6)]
    cm, idx, cells, proofs = _items(bundle, pairs)
    assert _verify(ctx, setups, cm, idx, cells, proofs) is True

    def refused(want, match, cm=cm, idx=idx, cells=cells, proofs=proofs):
        with pytest.raises(eb.B200Error, match=match) as e:
            _verify(ctx, setups, cm, idx, cells, proofs)
        assert e.value.status == want

    for k, bad in ((4, 128), (2, 2 ** 64 - 1)):
        i = idx[:]
        i[k] = bad
        refused(2, f"cell {k}: index {bad} is not below 128", idx=i)
    c = cells[:]
    c[3] = c[3][:32 * 40] + bls.R.to_bytes(32, "big") + c[3][32 * 41:]
    refused(2, "cell 3, element 40", cells=c)
    x_ge_p = bytearray(bls.P.to_bytes(48, "big"))
    x_ge_p[0] |= 0x80
    no_c = bytearray(proofs[2])
    no_c[0] &= 0x7F
    not_sub = bls.compress(B.g1_random_point(7))
    for point, want in ((bytes(x_ge_p), 2), (bytes(no_c), 3), (not_sub, 3)):
        p = proofs[:]
        p[4] = point
        refused(want, "the proof of cell 4 ", proofs=p)
        # a commitment is named by the first cell that uses it: blob 1's is cell 1's, then cell 4's
        m = [point if x == cm[1] else x for x in cm]
        refused(want, "the commitment of cell 1 ", cm=m)
    g1, g2, _ = setups
    two = ctx.bls12_381_g2_bases_upload(g2_points[:192], 2)
    try:
        for a, b in ((g1, two), (g1, g1), (g2, g2), (g1, 999999), (999999, g2)):
            with pytest.raises(eb.B200Error) as e:
                ctx.kzg_verify_cells(a, b, cm, idx, cells, proofs)
            assert e.value.status == 4
    finally:
        ctx.bases_free(two)
    valid = ctypes.c_int(-1)
    ind = np.array(idx, dtype=np.uint64)
    blob = b"".join(cells)
    for args in ((None, ind.ctypes.data_as(ctypes.c_void_p), blob, b"".join(proofs)), (b"".join(cm), None, blob, b"".join(proofs)),
                 (b"".join(cm), ind.ctypes.data_as(ctypes.c_void_p), None, b"".join(proofs)),
                 (b"".join(cm), ind.ctypes.data_as(ctypes.c_void_p), blob, None)):
        assert _ffi.lib.b200zk_kzg_verify_cells(ctx._h, g1, g2, *args, len(idx), ctypes.byref(valid)) == 4
    assert valid.value == -1
    assert _ffi.lib.b200zk_kzg_verify_cells(ctx._h, g1, g2, None, None, None, None, 0, ctypes.byref(valid)) == 0 and valid.value == 1
    assert _verify(ctx, setups, [], [], [], []) is True
    # the context still answers after every refusal
    assert _verify(ctx, setups, cm, idx, cells, proofs) is True


def test_kzg_settings_agrees_with_context(ctx, setups, points, g2_points, bundle):
    pairs = [(b, c) for b in (2, 3, 4) for c in (0, 64, 127)]
    cm, idx, cells, proofs = _items(bundle, pairs)
    s = KzgSettings(ctx, points, g2_monomial=g2_points)
    try:
        assert s.verify_cells(cm, idx, cells, proofs) is True is _verify(ctx, setups, cm, idx, cells, proofs)
        wrong = proofs[:]
        wrong[0], wrong[1] = proofs[1], proofs[0]
        assert s.verify_cells(cm, idx, cells, wrong) is False is _verify(ctx, setups, cm, idx, cells, wrong)
        assert s.verify_cells([], [], [], []) is True
        with pytest.raises(ValueError):
            s.verify_cells(cm, idx, cells, proofs[:-1])
        with pytest.raises(ValueError):
            s.verify_cells(cm, [128] + idx[1:], cells, proofs)
        with pytest.raises(ValueError):
            s.verify_cells(cm, idx, cells, [bls.compress(B.g1_random_point(7))] + proofs[1:])
    finally:
        s.close()


def test_verify_then_recover(ctx, setups, bundle):
    _, cs, cells, proofs = bundle
    rng = random.Random(11)
    blob_ids = (0, 5, 12)
    given = {b: rng.sample(range(128), 64) for b in blob_ids}
    pairs = [(b, c) for b in blob_ids for c in given[b]]
    assert _verify(ctx, setups, *_items(bundle, pairs)) is True
    items = [(given[b], [cells[b][c] for c in given[b]]) for b in blob_ids]
    rec_cells, rec_proofs = ctx.kzg_recover_cells_and_cell_proofs(setups[2], items)
    assert rec_cells == [x for b in blob_ids for x in cells[b]] and rec_proofs == [x for b in blob_ids for x in proofs[b]]
    cm = [cs[b] for b in blob_ids for _ in range(128)]
    assert _verify(ctx, setups, cm, [c for _ in blob_ids for c in range(128)], rec_cells, rec_proofs) is True
