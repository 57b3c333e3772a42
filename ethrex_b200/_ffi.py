"""ctypes binding of libb200zk.so (include/b200zk.h) -- the Python twin of rust/b200zk-sys.

The product path has NO CPU fallback: if the shared library is missing this module raises at
import time, and if no CUDA device is present `Context()` raises `NoDeviceError`.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B200ZK_LIB") or os.path.join(_HERE, "libb200zk.so")  # B200ZK_LIB: A/B builds of the same ABI (experiments)

# status codes (include/b200zk.h; 0..3 = /root/reference/crates/guest-program/src/crypto/zisk.rs:144-172)
OK, OK_INFINITY, ERR_NOT_IN_FIELD, ERR_NOT_ON_CURVE, ERR_INVALID_ARG, ERR_CUDA, ERR_NO_DEVICE, ERR_OOM, ERR_UNSUPPORTED = range(9)

# flags
POINTS_BE = 1 << 0
SCALARS_BE = 1 << 1
SCALARS_MONT = 1 << 2
OUT_NATIVE = 1 << 3
NTT_INVERSE = 1 << 4
NTT_COSET = 1 << 5
NTT_CANONICAL = 1 << 6
NTT_BE = 1 << 7
G16_INPUTS_DEVICE = 1 << 8
G16_H_COEFFS = 1 << 9
SCALARS_RAW = 1 << 10
POINTS_COMPRESSED = 1 << 11
ECRECOVER_LOW_S = 1  # b200zk_secp256k1_ecrecover_batch: reject s > n/2 (EIP-2)

_vp, _sz, _u32, _u64, _int = C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint64, C.c_int
_ctx = C.c_void_p


class Groth16Pk(C.Structure):
    """struct b200zk_groth16_pk (include/b200zk.h): columns 0..4 = A_g1, B_g1, B_g2, L_g1, H_g1"""
    _fields_ = [("log_n", C.c_uint32), ("reserved", C.c_uint32), ("handle", C.c_uint64 * 5), ("count", C.c_uint64 * 5), ("offset", C.c_uint64 * 5)]


class Groth16Zk(C.Structure):
    """struct b200zk_groth16_zk (include/b200zk.h): key-term handles (G1 alpha, beta, delta; G2 beta, delta) and the
    blinding scalars r, s as canonical little-endian bytes below the group order"""
    _fields_ = [("g1_terms", C.c_uint64), ("g2_terms", C.c_uint64), ("r", C.c_uint8 * 32), ("s", C.c_uint8 * 32)]


# name -> (restype, argtypes); every symbol include/b200zk.h declares
SIGNATURES = {
    "b200zk_abi_version": (_int, []),
    "b200zk_device_count": (_int, []),
    "b200zk_init": (_int, [_int, C.POINTER(_ctx)]),
    "b200zk_destroy": (None, [_ctx]),
    "b200zk_strerror": (C.c_char_p, [_int]),
    "b200zk_last_error": (C.c_char_p, [_ctx]),
    "b200zk_launch_count": (_u64, [_ctx]),
    "b200zk_synchronize": (_int, [_ctx]),
    "b200zk_g1_msm": (_int, [_ctx, _vp, _vp, _sz, _u32, _vp]),
    "b200zk_g2_msm": (_int, [_ctx, _vp, _vp, _sz, _u32, _vp]),
    "b200zk_fr_ntt": (_int, [_ctx, _vp, _u32, _u32, _vp]),
    "b200zk_g1_bases_upload": (_int, [_ctx, _vp, _sz, _u32, C.POINTER(_u64)]),
    "b200zk_g2_bases_upload": (_int, [_ctx, _vp, _sz, _u32, C.POINTER(_u64)]),
    "b200zk_g1_bases_from_device": (_int, [_ctx, _vp, _sz, _vp, C.POINTER(_u64)]),
    "b200zk_g2_bases_from_device": (_int, [_ctx, _vp, _sz, _vp, C.POINTER(_u64)]),
    "b200zk_bases_precompute": (_int, [_ctx, _u64, _u32]),
    "b200zk_bases_free": (_int, [_ctx, _u64]),
    "b200zk_g1_msm_resident_device": (_int, [_ctx, _u64, _vp, _sz, _u32, _vp, _vp]),
    "b200zk_g2_msm_resident_device": (_int, [_ctx, _u64, _vp, _sz, _u32, _vp, _vp]),
    "b200zk_g1_msm_resident": (_int, [_ctx, _u64, _vp, _sz, _u32, _vp]),
    "b200zk_g2_msm_resident": (_int, [_ctx, _u64, _vp, _sz, _u32, _vp]),
    "b200zk_g1_msm_device": (_int, [_ctx, _vp, _vp, _sz, _u32, _vp, _vp]),
    "b200zk_g2_msm_device": (_int, [_ctx, _vp, _vp, _sz, _u32, _vp, _vp]),
    "b200zk_g1_msm_device_async": (_int, [_ctx, _vp, _vp, _sz, _u32, _vp, _vp]),
    "b200zk_g2_msm_device_async": (_int, [_ctx, _vp, _vp, _sz, _u32, _vp, _vp]),
    "b200zk_fr_ntt_device": (_int, [_ctx, _vp, _u32, _u32, _vp, _vp]),
    "b200zk_set_ntt_root": (_int, [_ctx, _vp]),
    "b200zk_ntt_root_preset": (_int, [_int, _vp]),
    "b200zk_groth16_commit": (_int, [_ctx, _vp, _vp, _vp, _vp, _vp, _u32, _vp, _vp, _vp]),
    "b200zk_groth16_commit_partial": (_int, [_ctx, _vp, _vp, _vp, _vp, _vp, _u32, _vp, _vp]),
    "b200zk_groth16_fold": (_int, [_ctx, _vp, _sz, _vp, _vp, _vp]),
    "b200zk_groth16_prove": (_int, [_ctx, _vp, _vp, _vp, _vp, _vp, _vp, _u32, _vp, _vp]),
    "b200zk_groth16_fold_zk": (_int, [_ctx, _vp, _vp, _sz, _vp, _vp]),
    "b200zk_g1_msm_partial_device": (_int, [_ctx, _vp, _vp, _sz, _u32, _vp, _vp]),
    "b200zk_g2_msm_partial_device": (_int, [_ctx, _vp, _vp, _sz, _u32, _vp, _vp]),
    "b200zk_g1_msm_partial_resident_device": (_int, [_ctx, _u64, _vp, _sz, _u32, _vp, _vp]),
    "b200zk_g2_msm_partial_resident_device": (_int, [_ctx, _u64, _vp, _sz, _u32, _vp, _vp]),
    "b200zk_g1_msm_partial_resident": (_int, [_ctx, _u64, _vp, _sz, _u32, _vp, _vp]),
    "b200zk_g2_msm_partial_resident": (_int, [_ctx, _u64, _vp, _sz, _u32, _vp, _vp]),
    "b200zk_g1_fold_partials_device": (_int, [_ctx, _vp, _sz, _u32, _vp, _vp]),
    "b200zk_g2_fold_partials_device": (_int, [_ctx, _vp, _sz, _u32, _vp, _vp]),
    "b200zk_field_to_mont_device": (_int, [_ctx, _vp, _sz, _int, _vp]),
    "b200zk_field_from_mont_device": (_int, [_ctx, _vp, _sz, _int, _vp]),
    "b200zk_field_mul_device": (_int, [_ctx, _vp, _vp, _vp, _sz, _int, _u32, _vp]),
    "b200zk_fr_quotient_device": (_int, [_ctx, _vp, _vp, _vp, _vp, _sz, _vp, _vp]),
    "b200zk_fr_random_device": (_int, [_ctx, _vp, _sz, _u64, _u64, _u32, _vp]),
    "b200zk_g1_chain_device": (_int, [_ctx, _vp, _sz, _sz, _vp, _vp, _vp]),
    "b200zk_g2_chain_device": (_int, [_ctx, _vp, _sz, _sz, _vp, _vp, _vp]),
    "b200zk_g1_check_device": (_int, [_ctx, _vp, _sz, _vp, C.POINTER(_sz)]),
    "b200zk_g2_check_device": (_int, [_ctx, _vp, _sz, _vp, C.POINTER(_sz)]),
    "b200zk_set_msm_window": (_int, [_ctx, _u32]),
    "b200zk_set_msm_chunks": (_int, [_ctx, _u32]),
    "b200zk_set_msm_pair_rounds": (_int, [_ctx, _int]),
    "b200zk_last_msm_phase_ms": (_int, [_ctx, C.POINTER(C.c_float)]),
    "b200zk_set_profiling": (_int, [_ctx, _int]),
    "b200zk_msm_multi_resident_device": (_int, [_ctx, _vp, _sz, _vp, _sz, _u32, _vp, _vp, _vp]),
    "b200zk_bls12_381_g1_bases_upload": (_int, [_ctx, _vp, _sz, _u32, C.POINTER(_u64)]),
    "b200zk_bls12_381_g1_msm_resident": (_int, [_ctx, _u64, _vp, _sz, _u32, _vp]),
    "b200zk_kzg_blob_to_commitment": (_int, [_ctx, _u64, _vp, _sz, _vp]),
    "b200zk_kzg_blob_to_commitment_and_proof": (_int, [_ctx, _u64, _vp, _sz, _vp, _vp]),
    "b200zk_kzg_compute_proof": (_int, [_ctx, _u64, _vp, _sz, _vp, _vp, _vp]),
    "b200zk_bls12_381_g2_bases_upload": (_int, [_ctx, _vp, _sz, _u32, C.POINTER(_u64)]),
    "b200zk_bls12_381_pairing_check_batch": (_int, [_ctx, _vp, _vp, _sz, _vp, _vp]),
    "b200zk_kzg_verify_proof_batch": (_int, [_ctx, _u64, _vp, _vp, _vp, _vp, _sz, _vp, _vp]),
    "b200zk_kzg_verify_blob_proof_batch": (_int, [_ctx, _u64, _vp, _vp, _vp, _sz, C.POINTER(_int)]),
    "b200zk_kzg_compute_cells": (_int, [_ctx, _vp, _sz, _vp]),
    "b200zk_kzg_blob_to_commitment_and_cell_proofs": (_int, [_ctx, _u64, _u64, _vp, _sz, _vp, _vp]),
    "b200zk_kzg_verify_cell_proof_batch": (_int, [_ctx, _u64, _u64, _vp, _vp, _vp, _sz, C.POINTER(_int)]),
    "b200zk_bls12_381_g1_add_batch": (_int, [_ctx, _vp, _vp, _sz, _vp, _vp]),
    "b200zk_bls12_381_g2_add_batch": (_int, [_ctx, _vp, _vp, _sz, _vp, _vp]),
    "b200zk_bls12_381_g1_msm_batch": (_int, [_ctx, _vp, _vp, _sz, _vp, _vp]),
    "b200zk_bls12_381_g2_msm_batch": (_int, [_ctx, _vp, _vp, _sz, _vp, _vp]),
    "b200zk_secp256k1_ecrecover_batch": (_int, [_ctx, _vp, _vp, _sz, _u32, _vp, _vp]),
    "b200zk_secp256r1_verify_batch": (_int, [_ctx, _vp, _sz, _vp]),
    "b200zk_bn254_g1_add_batch": (_int, [_ctx, _vp, _vp, _sz, _vp, _vp]),
    "b200zk_bn254_g1_mul_batch": (_int, [_ctx, _vp, _vp, _sz, _vp, _vp]),
    "b200zk_bn254_pairing_check_batch": (_int, [_ctx, _vp, _vp, _sz, _vp, _vp]),
}


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(make -C ethrex_b200/csrc). There is no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here = the library does not export what the header declares
        fn.restype = res
        fn.argtypes = args
    return lib


lib = _load()
