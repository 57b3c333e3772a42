//! Raw bindings to `libb200zk.so` -- one declaration per symbol of `include/b200zk.h`, in the style of the
//! reference's own C-ABI precedent (`crates/guest-program/src/crypto/zisk.rs:5-64`): caller-owned buffers,
//! plain pointers and sizes, small integer status codes.
//!
//! NOTE: the build image for this repository has no Rust toolchain; this crate is shipped as source and is
//! kept in lock-step with the header by `tests/test_abi.py`.
#![no_std]
#![allow(non_camel_case_types)]

use core::ffi::{c_char, c_int, c_void};

/// Opaque context (one per process per GPU).
#[repr(C)]
pub struct b200zk_ctx {
    _private: [u8; 0],
}

pub const B200ZK_ABI_VERSION: c_int = 2;

// status codes: 0..3 follow zisk.rs:144-172
pub const B200ZK_OK: c_int = 0;
pub const B200ZK_OK_INFINITY: c_int = 1;
pub const B200ZK_ERR_NOT_IN_FIELD: c_int = 2;
pub const B200ZK_ERR_NOT_ON_CURVE: c_int = 3;
pub const B200ZK_ERR_INVALID_ARG: c_int = 4;
pub const B200ZK_ERR_CUDA: c_int = 5;
pub const B200ZK_ERR_NO_DEVICE: c_int = 6;
pub const B200ZK_ERR_OOM: c_int = 7;
pub const B200ZK_ERR_UNSUPPORTED: c_int = 8;

// flags
pub const B200ZK_POINTS_BE: u32 = 1 << 0;
pub const B200ZK_SCALARS_BE: u32 = 1 << 1;
pub const B200ZK_SCALARS_MONT: u32 = 1 << 2;
pub const B200ZK_OUT_NATIVE: u32 = 1 << 3;
pub const B200ZK_NTT_INVERSE: u32 = 1 << 4;
pub const B200ZK_NTT_COSET: u32 = 1 << 5;
pub const B200ZK_NTT_CANONICAL: u32 = 1 << 6;
pub const B200ZK_NTT_BE: u32 = 1 << 7;
pub const B200ZK_G16_INPUTS_DEVICE: u32 = 1 << 8;
pub const B200ZK_G16_H_COEFFS: u32 = 1 << 9;
pub const B200ZK_SCALARS_RAW: u32 = 1 << 10;
pub const B200ZK_POINTS_COMPRESSED: u32 = 1 << 11;
/// b200zk_secp256k1_ecrecover_batch: reject s > n/2 with status 2 (EIP-2, `Crypto::recover_signer`)
pub const B200ZK_ECRECOVER_LOW_S: u32 = 1;

/// `struct b200zk_groth16_pk` (include/b200zk.h): columns 0..4 = A_g1, B_g1 (handle 0 = absent), B_g2, L_g1, H_g1.
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct b200zk_groth16_pk {
    pub log_n: u32,
    pub reserved: u32,
    pub handle: [u64; 5],
    pub count: [u64; 5],
    pub offset: [u64; 5],
}

/// `struct b200zk_groth16_zk` (include/b200zk.h): resident handles of the key terms (G1: alpha, beta, delta; G2: beta,
/// delta; plain bases) and the blinding scalars r, s (canonical little-endian, below the group order).
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct b200zk_groth16_zk {
    pub g1_terms: u64,
    pub g2_terms: u64,
    pub r: [u8; 32],
    pub s: [u8; 32],
}

unsafe extern "C" {
    pub fn b200zk_abi_version() -> c_int;
    pub fn b200zk_device_count() -> c_int;
    pub fn b200zk_init(device: c_int, out: *mut *mut b200zk_ctx) -> c_int;
    pub fn b200zk_destroy(ctx: *mut b200zk_ctx);
    pub fn b200zk_strerror(status: c_int) -> *const c_char;
    pub fn b200zk_last_error(ctx: *const b200zk_ctx) -> *const c_char;
    pub fn b200zk_launch_count(ctx: *const b200zk_ctx) -> u64;
    pub fn b200zk_synchronize(ctx: *mut b200zk_ctx) -> c_int;

    pub fn b200zk_g1_msm(ctx: *mut b200zk_ctx, points: *const c_void, scalars: *const c_void, n: usize, flags: u32, out: *mut u8) -> c_int;
    pub fn b200zk_g2_msm(ctx: *mut b200zk_ctx, points: *const c_void, scalars: *const c_void, n: usize, flags: u32, out: *mut u8) -> c_int;
    pub fn b200zk_fr_ntt(ctx: *mut b200zk_ctx, data: *mut c_void, log_n: u32, flags: u32, coset_gen: *const u8) -> c_int;

    pub fn b200zk_g1_bases_upload(ctx: *mut b200zk_ctx, points: *const c_void, n: usize, flags: u32, handle: *mut u64) -> c_int;
    pub fn b200zk_g2_bases_upload(ctx: *mut b200zk_ctx, points: *const c_void, n: usize, flags: u32, handle: *mut u64) -> c_int;
    pub fn b200zk_g1_bases_from_device(ctx: *mut b200zk_ctx, d_points: *const c_void, n: usize, stream: *mut c_void, handle: *mut u64) -> c_int;
    pub fn b200zk_g2_bases_from_device(ctx: *mut b200zk_ctx, d_points: *const c_void, n: usize, stream: *mut c_void, handle: *mut u64) -> c_int;
    pub fn b200zk_bases_precompute(ctx: *mut b200zk_ctx, handle: u64, window_bits: u32) -> c_int;
    pub fn b200zk_bases_free(ctx: *mut b200zk_ctx, handle: u64) -> c_int;
    pub fn b200zk_g1_msm_resident_device(ctx: *mut b200zk_ctx, handle: u64, d_scalars: *const c_void, n: usize, flags: u32, stream: *mut c_void, out: *mut u8) -> c_int;
    pub fn b200zk_g2_msm_resident_device(ctx: *mut b200zk_ctx, handle: u64, d_scalars: *const c_void, n: usize, flags: u32, stream: *mut c_void, out: *mut u8) -> c_int;
    pub fn b200zk_g1_msm_resident(ctx: *mut b200zk_ctx, handle: u64, scalars: *const c_void, n: usize, flags: u32, out: *mut u8) -> c_int;
    pub fn b200zk_g2_msm_resident(ctx: *mut b200zk_ctx, handle: u64, scalars: *const c_void, n: usize, flags: u32, out: *mut u8) -> c_int;

    pub fn b200zk_g1_msm_device(ctx: *mut b200zk_ctx, d_points: *const c_void, d_scalars: *const c_void, n: usize, flags: u32, stream: *mut c_void, out: *mut u8) -> c_int;
    pub fn b200zk_g2_msm_device(ctx: *mut b200zk_ctx, d_points: *const c_void, d_scalars: *const c_void, n: usize, flags: u32, stream: *mut c_void, out: *mut u8) -> c_int;
    pub fn b200zk_g1_msm_device_async(ctx: *mut b200zk_ctx, d_points: *const c_void, d_scalars: *const c_void, n: usize, flags: u32, stream: *mut c_void, d_out68: *mut c_void) -> c_int;
    pub fn b200zk_g2_msm_device_async(ctx: *mut b200zk_ctx, d_points: *const c_void, d_scalars: *const c_void, n: usize, flags: u32, stream: *mut c_void, d_out132: *mut c_void) -> c_int;
    pub fn b200zk_fr_ntt_device(ctx: *mut b200zk_ctx, d_data: *mut c_void, log_n: u32, flags: u32, coset_gen: *const u8, stream: *mut c_void) -> c_int;
    pub fn b200zk_set_ntt_root(ctx: *mut b200zk_ctx, root_le: *const u8) -> c_int;
    pub fn b200zk_ntt_root_preset(preset: c_int, root_le_out: *mut u8) -> c_int;
    pub fn b200zk_groth16_commit(ctx: *mut b200zk_ctx, pk: *const b200zk_groth16_pk, witness: *const c_void, a_evals: *mut c_void, b_evals: *mut c_void, c_evals: *mut c_void, flags: u32, stream: *mut c_void, proof: *mut u8, b_g1: *mut u8) -> c_int;
    pub fn b200zk_groth16_commit_partial(ctx: *mut b200zk_ctx, pk: *const b200zk_groth16_pk, witness: *const c_void, a_evals: *mut c_void, b_evals: *mut c_void, c_evals: *mut c_void, flags: u32, stream: *mut c_void, d_partials768: *mut c_void) -> c_int;
    pub fn b200zk_groth16_fold(ctx: *mut b200zk_ctx, d_partials: *const c_void, count: usize, stream: *mut c_void, proof: *mut u8, b_g1: *mut u8) -> c_int;
    pub fn b200zk_groth16_prove(ctx: *mut b200zk_ctx, pk: *const b200zk_groth16_pk, zk: *const b200zk_groth16_zk, witness: *const c_void, a_evals: *mut c_void, b_evals: *mut c_void, c_evals: *mut c_void, flags: u32, stream: *mut c_void, proof: *mut u8) -> c_int;
    pub fn b200zk_groth16_fold_zk(ctx: *mut b200zk_ctx, zk: *const b200zk_groth16_zk, d_partials: *const c_void, count: usize, stream: *mut c_void, proof: *mut u8) -> c_int;
    // Groth16 from circom artifacts: a snarkjs .zkey loaded once, each .wtns witness proved in one call
    pub fn b200zk_groth16_zkey_load(ctx: *mut b200zk_ctx, zkey: *const c_void, len: usize, precompute: c_int, key: *mut u64) -> c_int;
    pub fn b200zk_groth16_zkey_free(ctx: *mut b200zk_ctx, key: u64) -> c_int;
    pub fn b200zk_groth16_zkey_info(ctx: *mut b200zk_ctx, key: u64, n_vars: *mut u32, n_public: *mut u32, log_n: *mut u32, vk: *mut u8, vk_len: usize) -> c_int;
    pub fn b200zk_groth16_zkey_prove(ctx: *mut b200zk_ctx, key: u64, wtns: *const c_void, len: usize, r: *const u8, s: *const u8, stream: *mut c_void, proof: *mut u8) -> c_int;
    pub fn b200zk_groth16_verify_batch(ctx: *mut b200zk_ctx, vk: *const u8, vk_len: usize, proofs: *const u8, public_inputs: *const u8, count: usize, valid: *mut u8, status: *mut u8, batch_ok: *mut c_int) -> c_int;
    // PLONK from circom artifacts: a snarkjs 0.7 PLONK .zkey loaded once, each .wtns witness proved in one call
    pub fn b200zk_plonk_zkey_load(ctx: *mut b200zk_ctx, zkey: *const c_void, len: usize, precompute: c_int, key: *mut u64) -> c_int;
    pub fn b200zk_plonk_zkey_free(ctx: *mut b200zk_ctx, key: u64) -> c_int;
    pub fn b200zk_plonk_zkey_info(ctx: *mut b200zk_ctx, key: u64, n_vars: *mut u32, n_public: *mut u32, log_n: *mut u32, vk: *mut u8, vk_len: usize) -> c_int;
    pub fn b200zk_plonk_zkey_prove(ctx: *mut b200zk_ctx, key: u64, wtns: *const c_void, len: usize, blinding: *const u8, stream: *mut c_void, proof: *mut u8) -> c_int;
    pub fn b200zk_plonk_last_round_ms(ctx: *mut b200zk_ctx, out_ms: *mut f32) -> c_int;

    pub fn b200zk_g1_msm_partial_device(ctx: *mut b200zk_ctx, d_points: *const c_void, d_scalars: *const c_void, n: usize, flags: u32, stream: *mut c_void, d_partial128: *mut c_void) -> c_int;
    pub fn b200zk_g2_msm_partial_device(ctx: *mut b200zk_ctx, d_points: *const c_void, d_scalars: *const c_void, n: usize, flags: u32, stream: *mut c_void, d_partial256: *mut c_void) -> c_int;
    pub fn b200zk_g1_msm_partial_resident_device(ctx: *mut b200zk_ctx, handle: u64, d_scalars: *const c_void, n: usize, flags: u32, stream: *mut c_void, d_partial128: *mut c_void) -> c_int;
    pub fn b200zk_g2_msm_partial_resident_device(ctx: *mut b200zk_ctx, handle: u64, d_scalars: *const c_void, n: usize, flags: u32, stream: *mut c_void, d_partial256: *mut c_void) -> c_int;
    pub fn b200zk_g1_msm_partial_resident(ctx: *mut b200zk_ctx, handle: u64, scalars: *const c_void, n: usize, flags: u32, stream: *mut c_void, d_partial128: *mut c_void) -> c_int;
    pub fn b200zk_g2_msm_partial_resident(ctx: *mut b200zk_ctx, handle: u64, scalars: *const c_void, n: usize, flags: u32, stream: *mut c_void, d_partial256: *mut c_void) -> c_int;
    pub fn b200zk_g1_fold_partials_device(ctx: *mut b200zk_ctx, d_partials: *const c_void, count: usize, flags: u32, stream: *mut c_void, out: *mut u8) -> c_int;
    pub fn b200zk_g2_fold_partials_device(ctx: *mut b200zk_ctx, d_partials: *const c_void, count: usize, flags: u32, stream: *mut c_void, out: *mut u8) -> c_int;

    pub fn b200zk_field_to_mont_device(ctx: *mut b200zk_ctx, d_data: *mut c_void, n: usize, which: c_int, stream: *mut c_void) -> c_int;
    pub fn b200zk_field_from_mont_device(ctx: *mut b200zk_ctx, d_data: *mut c_void, n: usize, which: c_int, stream: *mut c_void) -> c_int;
    pub fn b200zk_field_mul_device(ctx: *mut b200zk_ctx, d_a: *const c_void, d_b: *const c_void, d_out: *mut c_void, n: usize, which: c_int, repeat: u32, stream: *mut c_void) -> c_int;
    pub fn b200zk_fr_quotient_device(ctx: *mut b200zk_ctx, d_a: *const c_void, d_b: *const c_void, d_c: *const c_void, d_out: *mut c_void, n: usize, zinv: *const u8, stream: *mut c_void) -> c_int;
    pub fn b200zk_fr_random_device(ctx: *mut b200zk_ctx, d_out: *mut c_void, n: usize, seed: u64, start: u64, flags: u32, stream: *mut c_void) -> c_int;
    pub fn b200zk_g1_chain_device(ctx: *mut b200zk_ctx, d_out: *mut c_void, start: usize, n: usize, k: *const u8, d: *const u8, stream: *mut c_void) -> c_int;
    pub fn b200zk_g2_chain_device(ctx: *mut b200zk_ctx, d_out: *mut c_void, start: usize, n: usize, k: *const u8, d: *const u8, stream: *mut c_void) -> c_int;
    pub fn b200zk_g1_check_device(ctx: *mut b200zk_ctx, d_points: *const c_void, n: usize, stream: *mut c_void, bad_index: *mut usize) -> c_int;
    pub fn b200zk_g2_check_device(ctx: *mut b200zk_ctx, d_points: *const c_void, n: usize, stream: *mut c_void, bad_index: *mut usize) -> c_int;

    pub fn b200zk_set_msm_window(ctx: *mut b200zk_ctx, c: u32) -> c_int;
    pub fn b200zk_set_msm_chunks(ctx: *mut b200zk_ctx, chunks: u32) -> c_int;
    pub fn b200zk_last_msm_phase_ms(ctx: *mut b200zk_ctx, out_ms: *mut f32) -> c_int;
    pub fn b200zk_set_profiling(ctx: *mut b200zk_ctx, enabled: c_int) -> c_int;

    pub fn b200zk_msm_multi_resident_device(ctx: *mut b200zk_ctx, handles: *const u64, count: usize, d_scalars: *const c_void, n: usize, flags: u32, stream: *mut c_void, out: *mut u8, status: *mut c_int) -> c_int;
    pub fn b200zk_bls12_381_g1_bases_upload(ctx: *mut b200zk_ctx, points: *const c_void, n: usize, flags: u32, handle: *mut u64) -> c_int;
    pub fn b200zk_bls12_381_g1_msm_resident(ctx: *mut b200zk_ctx, handle: u64, scalars: *const c_void, n: usize, flags: u32, out: *mut u8) -> c_int;
    pub fn b200zk_kzg_blob_to_commitment(ctx: *mut b200zk_ctx, setup_handle: u64, blobs: *const u8, n_blobs: usize, commitments: *mut u8) -> c_int;
    pub fn b200zk_kzg_blob_to_commitment_and_proof(ctx: *mut b200zk_ctx, setup_handle: u64, blobs: *const u8, n_blobs: usize, commitments: *mut u8, proofs: *mut u8) -> c_int;
    pub fn b200zk_kzg_compute_proof(ctx: *mut b200zk_ctx, setup_handle: u64, blobs: *const u8, n_blobs: usize, z: *const u8, proofs: *mut u8, y: *mut u8) -> c_int;
    pub fn b200zk_bls12_381_g2_bases_upload(ctx: *mut b200zk_ctx, points: *const c_void, n: usize, flags: u32, handle: *mut u64) -> c_int;
    pub fn b200zk_bls12_381_pairing_check_batch(ctx: *mut b200zk_ctx, pairs: *const u8, pair_offsets: *const u32, count: usize, result: *mut u8, status: *mut u8) -> c_int;
    pub fn b200zk_kzg_verify_proof_batch(ctx: *mut b200zk_ctx, g2_setup: u64, commitments: *const u8, z: *const u8, y: *const u8, proofs: *const u8, n: usize, result: *mut u8, status: *mut u8) -> c_int;
    pub fn b200zk_kzg_verify_blob_proof_batch(ctx: *mut b200zk_ctx, g2_setup: u64, blobs: *const u8, commitments: *const u8, proofs: *const u8, n: usize, valid: *mut c_int) -> c_int;
    pub fn b200zk_kzg_compute_cells(ctx: *mut b200zk_ctx, blobs: *const u8, n_blobs: usize, cells: *mut u8) -> c_int;
    pub fn b200zk_kzg_blob_to_commitment_and_cell_proofs(ctx: *mut b200zk_ctx, g1_lagrange: u64, g1_monomial: u64, blobs: *const u8, n_blobs: usize, commitments: *mut u8, proofs: *mut u8) -> c_int;
    pub fn b200zk_kzg_verify_cell_proof_batch(ctx: *mut b200zk_ctx, g1_setup: u64, g2_setup: u64, blobs: *const u8, commitments: *const u8, proofs: *const u8, n_blobs: usize, valid: *mut c_int) -> c_int;
    pub fn b200zk_kzg_recover_cells_and_cell_proofs(ctx: *mut b200zk_ctx, g1_monomial: u64, cell_offsets: *const u32, cell_indices: *const u64, cells: *const u8, n_blobs: usize, cells_out: *mut u8, proofs_out: *mut u8) -> c_int;
    pub fn b200zk_kzg_verify_cells(ctx: *mut b200zk_ctx, g1_setup: u64, g2_setup: u64, commitments: *const u8, cell_indices: *const u64, cells: *const u8, proofs: *const u8, n_cells: usize, valid: *mut c_int) -> c_int;
    pub fn b200zk_bls12_381_g1_add_batch(ctx: *mut b200zk_ctx, a: *const u8, b: *const u8, count: usize, out: *mut u8, status: *mut u8) -> c_int;
    pub fn b200zk_bls12_381_g2_add_batch(ctx: *mut b200zk_ctx, a: *const u8, b: *const u8, count: usize, out: *mut u8, status: *mut u8) -> c_int;
    pub fn b200zk_bls12_381_g1_msm_batch(ctx: *mut b200zk_ctx, pairs: *const u8, pair_offsets: *const u32, count: usize, out: *mut u8, status: *mut u8) -> c_int;
    pub fn b200zk_bls12_381_g2_msm_batch(ctx: *mut b200zk_ctx, pairs: *const u8, pair_offsets: *const u32, count: usize, out: *mut u8, status: *mut u8) -> c_int;
    pub fn b200zk_bls12_381_map_fp_to_g1_batch(ctx: *mut b200zk_ctx, fps: *const u8, count: usize, out: *mut u8, status: *mut u8) -> c_int;
    pub fn b200zk_bls12_381_map_fp2_to_g2_batch(ctx: *mut b200zk_ctx, fp2s: *const u8, count: usize, out: *mut u8, status: *mut u8) -> c_int;
    pub fn b200zk_secp256k1_ecrecover_batch(ctx: *mut b200zk_ctx, sigs: *const u8, msgs: *const u8, count: usize, flags: u32, out: *mut u8, status: *mut u8) -> c_int;
    pub fn b200zk_secp256r1_verify_batch(ctx: *mut b200zk_ctx, inputs: *const u8, count: usize, result: *mut u8) -> c_int;
    pub fn b200zk_modexp_batch(ctx: *mut b200zk_ctx, data: *const u8, lens: *const u32, count: usize, out: *mut u8, status: *mut u8) -> c_int;
    pub fn b200zk_bn254_g1_add_batch(ctx: *mut b200zk_ctx, a: *const u8, b: *const u8, count: usize, out: *mut u8, status: *mut u8) -> c_int;
    pub fn b200zk_bn254_g1_mul_batch(ctx: *mut b200zk_ctx, points: *const u8, scalars: *const u8, count: usize, out: *mut u8, status: *mut u8) -> c_int;
    pub fn b200zk_bn254_pairing_check_batch(ctx: *mut b200zk_ctx, pairs: *const u8, pair_offsets: *const u32, count: usize, result: *mut u8, status: *mut u8) -> c_int;
}
