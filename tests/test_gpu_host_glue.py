"""The host glue every C entry point shares: resident handles refused by group, freed or unknown with each call's own
status and last_error text; tables built once per context or handle (one build launch on the first call, none after);
and the pair_offsets refusals of both pairing-check batches."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

import ethrex_b200 as eb  # noqa: E402
from ethrex_b200 import _ffi as F  # noqa: E402

BLOB = bytes(4096 * 32)
G1_ID = bytes([0xC0]) + bytes(47)  # compressed BLS12-381 identities: valid setup points
G2_ID = bytes([0xC0]) + bytes(95)
BN_GEN_BE = (1).to_bytes(32, "big") + (2).to_bytes(32, "big")  # the BN254 G1 generator


def _refused(ctx, call, text):
    with pytest.raises(eb.B200Error) as e:
        call()
    assert e.value.status == F.ERR_INVALID_ARG
    assert F.lib.b200zk_last_error(ctx._h).decode() == text


@pytest.fixture(scope="module")
def handles(ctx):
    h = {
        "bn254_g1": ctx.g1_bases_upload(BN_GEN_BE * 2, 2, F.POINTS_BE),
        "bn254_g2": ctx.g2_bases_upload(bytes(128 * 2), 2),
        "bls12_g1": ctx.bls12_381_g1_bases_upload(G1_ID * 2, 2),
        "bls12_g2": ctx.bls12_381_g2_bases_upload(G2_ID * 2, 2),
        "setup": ctx.bls12_381_g1_bases_upload(G1_ID * 4096, 4096),
    }
    freed = ctx.g1_bases_upload(BN_GEN_BE, 1, F.POINTS_BE)
    ctx.bases_free(freed)
    h["freed"] = freed
    h["unknown"] = max(h.values()) + 1000
    yield h
    for k in ("bn254_g1", "bn254_g2", "bls12_g1", "bls12_g2", "setup"):
        ctx.bases_free(h[k])


BAD = ["bn254_g1", "bn254_g2", "bls12_g1", "bls12_g2", "freed", "unknown"]


def _calls(ctx, h):
    """name -> (the group it accepts, call(handle), the refusal's last_error)"""
    d_sc = torch.zeros(8, dtype=torch.int32, device="cuda")
    d_part = torch.zeros(64, dtype=torch.int32, device="cuda")
    sc = bytes(32)
    g16 = lambda col: lambda bad: ctx.groth16_commit(  # noqa: E731
        ctx.groth16_pk(1, [bad if k == col else (h["bn254_g2"] if k == 2 else h["bn254_g1"]) for k in range(5)], [1] * 5, [0] * 5),
        bytes(32), bytes(64), bytes(64), bytes(64))
    cells = "kzg_blob_to_commitment_and_cell_proofs"
    return {
        "g1_msm_resident": ("bn254_g1", lambda b: ctx.g1_msm_resident(b, sc, 1), "msm_resident: unknown handle"),
        "g2_msm_resident": ("bn254_g2", lambda b: ctx.g2_msm_resident(b, sc, 1), "msm_resident: unknown handle"),
        "g1_msm_resident_device": ("bn254_g1", lambda b: ctx.g1_msm_resident_device(b, d_sc, 1), "msm_resident_device: unknown handle"),
        "g2_msm_resident_device": ("bn254_g2", lambda b: ctx.g2_msm_resident_device(b, d_sc, 1), "msm_resident_device: unknown handle"),
        "g1_msm_partial_resident": ("bn254_g1", lambda b: ctx.g1_msm_partial_resident(b, sc, 1, d_part), "msm_partial_resident: unknown handle"),
        "g2_msm_partial_resident": ("bn254_g2", lambda b: ctx.g2_msm_partial_resident(b, sc, 1, d_part), "msm_partial_resident: unknown handle"),
        "g1_msm_partial_resident_device": ("bn254_g1", lambda b: ctx.g1_msm_partial_resident_device(b, d_sc, 1, d_part),
                                           "msm_partial_resident: unknown handle"),
        "g2_msm_partial_resident_device": ("bn254_g2", lambda b: ctx.g2_msm_partial_resident_device(b, d_sc, 1, d_part),
                                           "msm_partial_resident: unknown handle"),
        "groth16_commit_a": ("bn254_g1", g16(0), "groth16_commit: unknown handle or wrong group for a column"),
        "groth16_commit_b2": ("bn254_g2", g16(2), "groth16_commit: unknown handle or wrong group for a column"),
        "bls12_381_g1_msm_resident": ("bls12_g1", lambda b: ctx.bls12_381_g1_msm_resident(b, sc, 1), "bls12_381_g1_msm_resident: unknown handle"),
        "kzg_blob_to_commitment": ("bls12_g1", lambda b: ctx.kzg_blob_to_commitment(b, BLOB), "kzg_blob_to_commitment: unknown setup handle"),
        "kzg_blob_to_commitment_and_proof": ("bls12_g1", lambda b: ctx.kzg_blob_to_commitment_and_proof(b, BLOB),
                                             "kzg_blob_to_commitment_and_proof: unknown setup handle"),
        "kzg_compute_proof": ("bls12_g1", lambda b: ctx.kzg_compute_proof(b, BLOB, bytes(32)), "kzg_compute_proof: unknown setup handle"),
        "kzg_verify_proof_batch": ("bls12_g2", lambda b: ctx.kzg_verify_proof_batch(b, G1_ID, bytes(32), bytes(32), G1_ID),
                                   "kzg_verify_proof_batch: unknown BLS12-381 G2 setup handle"),
        "kzg_verify_blob_proof_batch": ("bls12_g2", lambda b: ctx.kzg_verify_blob_proof_batch(b, BLOB, G1_ID, G1_ID),
                                        "kzg_verify_blob_proof_batch: unknown BLS12-381 G2 setup handle"),
        "kzg_verify_cell_proof_batch_g1": ("bls12_g1", lambda b: ctx.kzg_verify_cell_proof_batch(b, h["bls12_g2"], BLOB, G1_ID, G1_ID * 128),
                                           "kzg_verify_cell_proof_batch: unknown G1 setup handle"),
        "kzg_verify_cell_proof_batch_g2": ("bls12_g2", lambda b: ctx.kzg_verify_cell_proof_batch(h["setup"], b, BLOB, G1_ID, G1_ID * 128),
                                           "kzg_verify_cell_proof_batch: unknown BLS12-381 G2 setup handle"),
        "cell_proofs_lagrange": ("bls12_g1", lambda b: ctx.kzg_blob_to_commitment_and_cell_proofs(b, h["setup"], BLOB),
                                 f"{cells} (g1_lagrange): unknown setup handle"),
        "cell_proofs_monomial": ("bls12_g1", lambda b: ctx.kzg_blob_to_commitment_and_cell_proofs(h["setup"], b, BLOB),
                                 f"{cells} (g1_monomial): unknown setup handle"),
    }


def test_handle_group_matrix(ctx, handles):
    probe = lambda: ctx.g1_msm_resident(handles["bn254_g1"], (3).to_bytes(32, "little") * 2, 2)  # noqa: E731
    before = probe()
    assert before != bytes(64)
    for name, (group, call, text) in _calls(ctx, handles).items():
        for bad in BAD:
            if bad != group:
                _refused(ctx, lambda: call(handles[bad]), text)
    # calls that accept several groups: only freed and unknown handles, and the groups they reject by name
    d_sc = torch.zeros(8, dtype=torch.int32, device="cuda")
    for bad in ("freed", "unknown"):
        _refused(ctx, lambda: ctx.bases_precompute(handles[bad]), "bases_precompute: unknown handle")
        _refused(ctx, lambda: ctx.bases_free(handles[bad]), "bases_free: unknown handle")
        _refused(ctx, lambda: ctx.msm_multi_resident_device([handles[bad]], [False], d_sc, 1), "msm_multi_resident_device: unknown handle")
    _refused(ctx, lambda: ctx.bases_precompute(handles["bls12_g2"]), "bases_precompute: BLS12-381 G2 handles are pairing inputs, not MSM bases")
    for bad in ("bls12_g1", "bls12_g2"):
        _refused(ctx, lambda: ctx.msm_multi_resident_device([handles["bn254_g1"], handles[bad]], [False, False], d_sc, 1),
                 "msm_multi_resident_device: BLS12-381 bases in a BN254 call")
    assert probe() == before


@pytest.fixture
def fresh(ctx):
    """a new Context, none of its tables built yet"""
    with eb.Context(0) as c:
        yield c


def _launches(ctx, call):
    n0 = ctx.launch_count
    out = call()
    return ctx.launch_count - n0, out


@pytest.mark.parametrize("which", ["secp256k1_ecrecover_batch", "secp256r1_verify_batch", "kzg_compute_proof", "kzg_compute_cells"])
def test_table_built_once_per_context(fresh, which):
    c = fresh
    setup = c.bls12_381_g1_bases_upload(G1_ID * 4096, 4096) if which == "kzg_compute_proof" else None
    call = {
        "secp256k1_ecrecover_batch": lambda: c.secp256k1_ecrecover_batch(bytes(range(65)) * 3, bytes(range(32)) * 3),
        "secp256r1_verify_batch": lambda: c.secp256r1_verify_batch(bytes(range(160)) * 3),
        "kzg_compute_proof": lambda: c.kzg_compute_proof(setup, BLOB, (5).to_bytes(32, "big")),
        "kzg_compute_cells": lambda: c.kzg_compute_cells(BLOB),
    }[which]
    first, out1 = _launches(c, call)
    second, out2 = _launches(c, call)
    assert first - second == 1  # the table's build kernel
    assert out1 == out2


def test_fk20_table_built_once_per_handle(fresh):
    c = fresh
    lag = c.bls12_381_g1_bases_upload(G1_ID * 4096, 4096)
    c.kzg_compute_cells(BLOB)  # the context's cell twiddles, built before the handle's first cell-proof call
    for _ in range(2):  # a fresh monomial handle, then the same after bases_free and a re-upload
        mono = c.bls12_381_g1_bases_upload(G1_ID * 4096, 4096)
        call = lambda: c.kzg_blob_to_commitment_and_cell_proofs(lag, mono, BLOB)  # noqa: E731
        first, out1 = _launches(c, call)
        second, out2 = _launches(c, call)
        assert first - second == 1  # the FK20 table's build kernel
        assert out1 == out2
        c.bases_free(mono)


@pytest.mark.parametrize("fn,what,pair", [("b200zk_bn254_pairing_check_batch", "pairing_check_batch", 192),
                                          ("b200zk_bls12_381_pairing_check_batch", "bls12_381_pairing_check_batch", 384)])
def test_pair_offsets_refused(ctx, fn, what, pair):
    check = getattr(F.lib, fn)
    pairs = C.create_string_buffer(2 * pair)
    res, st = C.create_string_buffer(2), C.create_string_buffer(2)

    def offs(*v):
        return (C.c_uint32 * len(v))(*v)
    assert check(ctx._h, pairs, offs(1, 1), 1, res, st) == F.ERR_INVALID_ARG
    assert F.lib.b200zk_last_error(ctx._h).decode() == f"{what}: pair_offsets[0] must be 0"
    assert check(ctx._h, pairs, offs(0, 2, 1), 2, res, st) == F.ERR_INVALID_ARG
    assert F.lib.b200zk_last_error(ctx._h).decode() == f"{what}: pair_offsets must be non-decreasing"
    assert check(ctx._h, None, offs(0, 0), 1, res, st) == F.OK  # an empty check still runs
