"""EIP-7594 cell recovery on the device (b200zk_kzg_recover_cells_and_cell_proofs) over the synthetic known-tau setup of
tests/test_gpu_kzg_cell_proofs.py.  From every pattern of given cells the call returns, byte for byte, the cells of
b200zk_kzg_compute_cells and the proofs of b200zk_kzg_blob_to_commitment_and_cell_proofs, which tests/kzg_cells_ref.py
checks in turn; malformed or inconsistent input gets its status and leaves the outputs untouched."""
import ctypes

import numpy as np
import pytest

import bls_ref as bls
import kzg_cells_ref as cells_ref
import kzg_recover_ref as ref
import kzg_ref

pytestmark = pytest.mark.gpu

import ethrex_b200 as eb  # noqa: E402
from ethrex_b200 import _ffi  # noqa: E402
from ethrex_b200.kzg import KzgSettings  # noqa: E402

TAU = 0x2F1B7C93D4A5E6F708192A3B4C5D6E7F8091A2B3C4D5E6F708192A3B4C5D6E7F % bls.R
PATTERNS = ref.patterns(seed=7594)
NAMES = sorted(PATTERNS)


def _monomial_blob(e):
    return kzg_ref.to_blob([pow(w, e, bls.R) for w in kzg_ref.roots_brp()])


@pytest.fixture(scope="module")
def points():
    return b"".join(bls.compress(p) for p in bls.generator_multiples(bls.lagrange_setup_scalars(TAU)))


@pytest.fixture(scope="module")
def monomial():
    return b"".join(bls.compress(p) for p in bls.generator_multiples([pow(TAU, i, bls.R) for i in range(4096)]))


@pytest.fixture(scope="module")
def setups(ctx, points, monomial):
    lag = ctx.bls12_381_g1_bases_upload(points, 4096)
    mono = ctx.bls12_381_g1_bases_upload(monomial, 4096)
    yield lag, mono
    for h in (lag, mono):
        ctx.bases_free(h)


@pytest.fixture(scope="module")
def bundle(ctx, setups):
    """24 blobs (zero, all r - 1, X^4095, X^64, X^63, then random) with their 128 cells and 128 proofs each from the
    existing device calls; the first six are held against the oracle"""
    rng = np.random.default_rng(7594)
    blobs = [bytes(131072), kzg_ref.to_blob([bls.R - 1] * 4096), _monomial_blob(4095), _monomial_blob(64), _monomial_blob(63)]
    blobs += [kzg_ref.to_blob([int.from_bytes(rng.bytes(32), "big") % bls.R for _ in range(4096)]) for _ in range(19)]
    cells = ctx.kzg_compute_cells(b"".join(blobs))
    proofs = ctx.kzg_blob_to_commitment_and_cell_proofs(setups[0], setups[1], b"".join(blobs))[1]
    proofs = [proofs[128 * b:128 * (b + 1)] for b in range(len(blobs))]
    _, oracle_proofs = cells_ref.bundle(blobs[:6], TAU)
    for b in range(6):
        assert cells[b] == cells_ref.compute_cells(blobs[b])
        assert proofs[b] == oracle_proofs[128 * b:128 * (b + 1)]
    return blobs, cells, proofs


def _items(cells, blob_ids, names):
    return [(PATTERNS[n], [cells[b][c] for c in PATTERNS[n]]) for b, n in zip(blob_ids, names)]


def _expect(cells, proofs, blob_ids):
    return [c for b in blob_ids for c in cells[b]], [p for b in blob_ids for p in proofs[b]]


@pytest.mark.parametrize("name", NAMES)
def test_pattern_rebuilds_cells_and_proofs(ctx, setups, bundle, name):
    """one call of six blobs (every special blob and a random one), all given the same pattern"""
    _, cells, proofs = bundle
    ids = list(range(6))
    got = ctx.kzg_recover_cells_and_cell_proofs(setups[1], _items(cells, ids, [name] * 6))
    assert got == _expect(cells, proofs, ids)


@pytest.mark.parametrize("k", [1, 6, 24])
def test_mixed_batch_agrees_with_single_calls(ctx, setups, bundle, k):
    """k blobs in one call, a different pattern per blob; each also recovered alone"""
    _, cells, proofs = bundle
    ids = list(range(24))[-k:]
    names = [NAMES[(b * 7) % len(NAMES)] for b in ids]
    batch = ctx.kzg_recover_cells_and_cell_proofs(setups[1], _items(cells, ids, names))
    assert batch == _expect(cells, proofs, ids)
    for i, (b, n) in enumerate(zip(ids, names)):
        one = ctx.kzg_recover_cells_and_cell_proofs(setups[1], _items(cells, [b], [n]))
        assert one == (batch[0][128 * i:128 * (i + 1)], batch[1][128 * i:128 * (i + 1)])


def _raw(ctx, mono, items):
    """(status, last error, whether both output buffers are untouched) of a direct C call"""
    offsets = np.cumsum([0] + [len(ix) for ix, _ in items]).astype(np.uint32)
    ind = np.array([c for ix, _ in items for c in ix] or [0], dtype=np.uint64)
    data = np.frombuffer(b"".join(b"".join(cs) for _, cs in items) or b"\0", dtype=np.uint8)
    k = len(items)
    co, pr = bytearray(b"\xAA" * 262144 * k), bytearray(b"\xAA" * 6144 * k)
    st = _ffi.lib.b200zk_kzg_recover_cells_and_cell_proofs(ctx._h, mono, offsets.ctypes.data_as(ctypes.c_void_p),
                                                           ind.ctypes.data_as(ctypes.c_void_p), data.ctypes.data_as(ctypes.c_void_p), k,
                                                           (ctypes.c_char * len(co)).from_buffer(co), (ctypes.c_char * len(pr)).from_buffer(pr))
    return st, _ffi.lib.b200zk_last_error(ctx._h).decode(), co == b"\xAA" * len(co) and pr == b"\xAA" * len(pr)


def test_statuses(ctx, setups, bundle, monomial):
    _, cells, _ = bundle
    mono = setups[1]
    good = _items(cells, [5], ["random96"])[0]

    def with_blob1(ix, cs):
        return [good, (ix, cs)]

    ix96, cs96 = good
    cases = {
        "63 cells": (with_blob1(ix96[:63], cs96[:63]), 2, "blob 1 has 63 cells"),
        "129 cells": (with_blob1(list(range(128)) + [0], [cells[6][c] for c in range(128)] + [cells[6][0]]), 2, "blob 1 has 129 cells"),
        "repeated index": (with_blob1(ix96[:70] + [ix96[3]], cs96[:70] + [cs96[3]]), 2, "blob 1, cell 70: index %d is repeated" % ix96[3]),
        "index 128": (with_blob1(ix96[:64] + [128], cs96[:65]), 2, "blob 1, cell 64: index 128 is not below 128"),
        "element r": (with_blob1(ix96, cs96[:10] + [cs96[10][:32 * 5] + bls.R.to_bytes(32, "big") + cs96[10][32 * 6:]] + cs96[11:]), 2,
                      "blob 1, cell 10, element 5 is >="),
        "corrupt 65th": (with_blob1(ix96[:65], cs96[:64] + [cs96[64][:-1] + bytes([cs96[64][-1] ^ 1])]), 3,
                         "blob 1, cell 64 (index %d) does not lie" % ix96[64]),
    }
    for name, (items, status, msg) in cases.items():
        st, err, untouched = _raw(ctx, mono, items)
        assert (st, untouched) == (status, True), name
        assert msg in err, (name, err)
    # a consistent input with more than 64 cells passes the same check
    assert _raw(ctx, mono, [good])[0] == 0
    with pytest.raises(eb.B200Error) as e:
        ctx.kzg_recover_cells_and_cell_proofs(mono, [(ix96[:65], cs96[:64] + [cs96[65]])])
    assert e.value.status == 3


def test_handles(ctx, setups, bundle, monomial):
    _, cells, _ = bundle
    items = _items(cells, [7], ["odd"])
    g2 = ctx.bls12_381_g2_bases_upload(cells_ref.g2_setup(TAU)[:96 * 2], 2)
    small = ctx.bls12_381_g1_bases_upload(monomial[:48 * 4095], 4095)
    freed = ctx.bls12_381_g1_bases_upload(monomial, 4096)
    ctx.bases_free(freed)
    try:
        for h in (g2, small, freed, 999999):
            st, _, untouched = _raw(ctx, h, items)
            assert (st, untouched) == (4, True)
    finally:
        ctx.bases_free(g2)
        ctx.bases_free(small)
    assert ctx.kzg_recover_cells_and_cell_proofs(setups[1], []) == ([], [])


def test_kzg_settings_agrees_with_context(ctx, setups, points, monomial, bundle):
    _, cells, proofs = bundle
    items = _items(cells, [8, 9], ["even", "random127"])
    want = ctx.kzg_recover_cells_and_cell_proofs(setups[1], items)
    s = KzgSettings(ctx, points, precompute=False, g1_monomial=monomial)
    try:
        got_cells, got_proofs = s.recover_cells_and_kzg_proofs_batch(items)
        assert [c for b in got_cells for c in b] == want[0] and [p for b in got_proofs for p in b] == want[1]
        assert s.recover_cells_and_kzg_proofs(*items[1]) == (cells[9], proofs[9])
        assert s.recover_cells_and_kzg_proofs_batch([]) == ([], [])
        ix, cs = items[0]
        with pytest.raises(ValueError):
            s.recover_cells_and_kzg_proofs(ix[:63], cs[:63])
        with pytest.raises(ValueError):
            s.recover_cells_and_kzg_proofs(ix[:65], cs[:64] + [cs[0]])  # status 3
    finally:
        s.close()
    plain = KzgSettings(ctx, points, precompute=False)
    try:
        with pytest.raises(ValueError, match="g1_monomial"):
            plain.recover_cells_and_kzg_proofs(*items[0])
    finally:
        plain.close()
