//! `B200Crypto`: the three BN254 calls of the reference's `Crypto` trait
//! (`crates/common/crypto/provider.rs:201-330`), its EIP-2537 G1/G2 addition and MSM (`provider.rs:549-640`) and its
//! BLS12-381 pairing check (`provider.rs:642-672`), its secp256k1 signer recovery (`provider.rs:63-171`) and its P-256
//! signature verification (`provider.rs:415-459`) on the GPU.  The trait is one item per call; a provider that wants
//! throughput collects the items of a block (or of the batch being proved) and calls the `*_batch` wrappers of
//! [`crate::ffi::B200zk`] directly -- the single-item methods below are the drop-in form.
//!
//! Error mapping follows the reference: the levm wrappers reject coordinates >= p before the curve call
//! (`crates/vm/levm/src/precompiles.rs:801-820`, `PrecompileError::CoordinateExceedsFieldModulus`), the provider
//! reports points off the curve as `CryptoError::InvalidPoint`.
use ethrex_common::Address;
use ethrex_crypto::{Crypto, CryptoError};

use crate::ffi::{global, ItemStatus, RecoverStatus};

#[derive(Debug, Default, Clone, Copy)]
pub struct B200Crypto;

fn device_error<E: std::fmt::Display>(e: E) -> CryptoError {
    CryptoError::Other(e.to_string())
}

fn item_error(status: ItemStatus, what: &'static str) -> CryptoError {
    match status {
        ItemStatus::NotInField => CryptoError::InvalidInput("coordinate exceeds the field modulus"),
        _ => CryptoError::InvalidPoint(what),
    }
}

fn recover_error(status: RecoverStatus) -> CryptoError {
    match status {
        RecoverStatus::InvalidSignature => CryptoError::InvalidSignature,
        RecoverStatus::RecoveryFailed => CryptoError::RecoveryFailed,
        RecoverStatus::InvalidRecoveryId => CryptoError::InvalidRecoveryId,
        other => CryptoError::Other(format!("b200zk ecrecover status {other:?}")),
    }
}

/// keccak256 of each recovered public key, one device call for all items
fn ecrecover_batch(items: &[([u8; 65], [u8; 32])], low_s: bool) -> Result<Vec<Result<[u8; 32], CryptoError>>, CryptoError> {
    let mut sigs = Vec::with_capacity(items.len().saturating_mul(65));
    let mut msgs = Vec::with_capacity(items.len().saturating_mul(32));
    for (sig, msg) in items {
        sigs.extend_from_slice(sig);
        msgs.extend_from_slice(msg);
    }
    let mut gpu = global().map_err(device_error)?.lock().map_err(device_error)?;
    let res = gpu.secp256k1_ecrecover_batch(&sigs, &msgs, low_s).map_err(device_error)?;
    Ok(res.into_iter().map(|r| r.map_err(recover_error)).collect())
}

fn address_of(hash: &[u8; 32]) -> Address {
    Address::from_slice(hash.split_at(12).1)
}

/// Transaction senders in one device call: the drop-in for the `par_iter` of `Block::get_transactions_with_sender`
/// (`crates/common/types/block.rs:323-333`).  Each item is what `Crypto::recover_signer` takes (a 65-byte r | s | recid
/// signature and the 32-byte signing hash), with its EIP-2 low-s rule; the results are in item order.
pub fn recover_signers_batch(items: &[([u8; 65], [u8; 32])]) -> Vec<Result<Address, CryptoError>> {
    match ecrecover_batch(items, true) {
        Ok(res) => res.into_iter().map(|r| r.map(|h| address_of(&h))).collect(),
        Err(e) => items.iter().map(|_| Err(CryptoError::Other(e.to_string()))).collect(),
    }
}

/// P256VERIFY (EIP-7951) for a block's calls in one device call.  Each item is what `Crypto::secp256r1_verify` takes:
/// the 32-byte message hash, r | s and qx | qy; the results are in item order.  The trait has no error channel, so a
/// device error makes every item `false`.
pub fn verify_p256_batch(items: &[([u8; 32], [u8; 64], [u8; 64])]) -> Vec<bool> {
    let mut inputs = Vec::with_capacity(items.len().saturating_mul(160));
    for (msg, sig, pk) in items {
        inputs.extend_from_slice(msg);
        inputs.extend_from_slice(sig);
        inputs.extend_from_slice(pk);
    }
    let res = global()
        .map_err(device_error)
        .and_then(|g| g.lock().map_err(device_error))
        .and_then(|mut gpu| gpu.secp256r1_verify_batch(&inputs).map_err(device_error));
    match res {
        Ok(v) if v.len() == items.len() => v,
        _ => vec![false; items.len()],
    }
}

impl Crypto for B200Crypto {
    /// The rules and their order are in include/b200zk.h (p256's `verify_prehash` as the reference calls it, EIP-7951).
    fn secp256r1_verify(&self, msg: &[u8; 32], sig: &[u8; 64], pk: &[u8; 64]) -> bool {
        verify_p256_batch(&[(*msg, *sig, *pk)]).first().copied().unwrap_or(false)
    }

    /// Follows the reference's default (libsecp256k1) path, recids 2 and 3 included; see include/b200zk.h.
    fn secp256k1_ecrecover(&self, sig: &[u8; 64], recid: u8, msg: &[u8; 32]) -> Result<[u8; 32], CryptoError> {
        let mut full = [0u8; 65];
        let (head, tail) = full.split_at_mut(64);
        head.copy_from_slice(sig);
        tail.copy_from_slice(&[recid]);
        ecrecover_batch(&[(full, *msg)], false)?
            .into_iter()
            .next()
            .unwrap_or_else(|| Err(CryptoError::Other("b200zk returned no result".to_string())))
    }

    fn recover_signer(&self, sig: &[u8; 65], msg: &[u8; 32]) -> Result<Address, CryptoError> {
        recover_signers_batch(&[(*sig, *msg)])
            .into_iter()
            .next()
            .unwrap_or_else(|| Err(CryptoError::Other("b200zk returned no result".to_string())))
    }

    fn bn254_g1_add(&self, p1: &[u8], p2: &[u8]) -> Result<[u8; 64], CryptoError> {
        let (a, b) = (p1.get(..64).ok_or(CryptoError::InvalidInput("G1 point must be 64 bytes"))?, p2.get(..64).ok_or(CryptoError::InvalidInput("G1 point must be 64 bytes"))?);
        let mut gpu = global().map_err(device_error)?.lock().map_err(device_error)?;
        let (out, st) = gpu.bn254_g1_add_batch(a, b).map_err(device_error)?;
        match st.first().copied() {
            Some(ItemStatus::Ok | ItemStatus::OkIdentity) => <[u8; 64]>::try_from(out.as_slice()).map_err(device_error),
            Some(bad) => Err(item_error(bad, "G1 point not on curve")),
            None => Err(CryptoError::Other("b200zk returned no status".to_string())),
        }
    }

    fn bn254_g1_mul(&self, point: &[u8], scalar: &[u8]) -> Result<[u8; 64], CryptoError> {
        let (p, k) = (point.get(..64).ok_or(CryptoError::InvalidInput("invalid input length"))?, scalar.get(..32).ok_or(CryptoError::InvalidInput("invalid input length"))?);
        let mut gpu = global().map_err(device_error)?.lock().map_err(device_error)?;
        let (out, st) = gpu.bn254_g1_mul_batch(p, k).map_err(device_error)?;
        match st.first().copied() {
            Some(ItemStatus::Ok | ItemStatus::OkIdentity) => <[u8; 64]>::try_from(out.as_slice()).map_err(device_error),
            Some(bad) => Err(item_error(bad, "G1 point not on curve")),
            None => Err(CryptoError::Other("b200zk returned no status".to_string())),
        }
    }

    fn bn254_pairing_check(&self, pairs: &[(&[u8], &[u8])]) -> Result<bool, CryptoError> {
        let mut calldata = Vec::with_capacity(pairs.len().saturating_mul(192));
        for (g1, g2) in pairs {
            calldata.extend_from_slice(g1.get(..64).ok_or(CryptoError::InvalidInput("G1 must be 64 bytes"))?);
            calldata.extend_from_slice(g2.get(..128).ok_or(CryptoError::InvalidInput("G2 must be 128 bytes"))?);
        }
        let mut gpu = global().map_err(device_error)?.lock().map_err(device_error)?;
        let res = gpu.bn254_pairing_check_batch(&[calldata.as_slice()]).map_err(device_error)?;
        match res.first() {
            Some(Ok(v)) => Ok(*v),
            Some(Err(bad)) => Err(item_error(*bad, "G1/G2 not on BN254 curve")),
            None => Err(CryptoError::Other("b200zk returned no result".to_string())),
        }
    }

    /// The trait passes 48-byte big-endian coordinates (G2: x.c0, x.c1, y.c0, y.c1); the device call takes the EIP-2537
    /// 64-byte form, so each is re-padded with 16 leading zero bytes.  No setup is needed.
    fn bls12_381_pairing_check(&self, pairs: &[(([u8; 48], [u8; 48]), ([u8; 48], [u8; 48], [u8; 48], [u8; 48]))]) -> Result<bool, CryptoError> {
        let mut calldata = Vec::with_capacity(pairs.len().saturating_mul(384));
        for ((x, y), (x0, x1, y0, y1)) in pairs {
            for fp in [x, y, x0, x1, y0, y1] {
                calldata.extend_from_slice(&[0u8; 16]);
                calldata.extend_from_slice(fp);
            }
        }
        let mut gpu = global().map_err(device_error)?.lock().map_err(device_error)?;
        let res = gpu.bls12_381_pairing_check_batch(&[calldata.as_slice()]).map_err(device_error)?;
        match res.first() {
            Some(Ok(v)) => Ok(*v),
            Some(Err(bad)) => Err(item_error(*bad, "G1/G2 not on the BLS12-381 curve or not in the subgroup")),
            None => Err(CryptoError::Other("b200zk returned no result".to_string())),
        }
    }

    fn bls12_381_g1_add(&self, a: ([u8; 48], [u8; 48]), b: ([u8; 48], [u8; 48])) -> Result<[u8; 96], CryptoError> {
        let (pa, pb) = (pad_g1(&a), pad_g1(&b));
        let mut gpu = global().map_err(device_error)?.lock().map_err(device_error)?;
        let (out, st) = gpu.bls12_381_g1_add_batch(&pa, &pb).map_err(device_error)?;
        match st.first().copied() {
            Some(ItemStatus::Ok | ItemStatus::OkIdentity) => Ok(unpad::<96>(&out)),
            Some(bad) => Err(item_error(bad, "G1 point not on curve")),
            None => Err(CryptoError::Other("b200zk returned no status".to_string())),
        }
    }

    fn bls12_381_g1_msm(&self, pairs: &[(([u8; 48], [u8; 48]), [u8; 32])]) -> Result<[u8; 96], CryptoError> {
        let mut calldata = Vec::with_capacity(pairs.len().saturating_mul(160));
        for (point, scalar) in pairs {
            calldata.extend_from_slice(&pad_g1(point));
            calldata.extend_from_slice(scalar);
        }
        let mut gpu = global().map_err(device_error)?.lock().map_err(device_error)?;
        let res = gpu.bls12_381_g1_msm_batch(&[calldata.as_slice()]).map_err(device_error)?;
        match res.first() {
            Some(Ok(out)) => Ok(unpad::<96>(out)),
            Some(Err(bad)) => Err(item_error(*bad, "G1 point not on curve or not in subgroup")),
            None => Err(CryptoError::Other("b200zk returned no result".to_string())),
        }
    }

    fn bls12_381_g2_add(&self, a: ([u8; 48], [u8; 48], [u8; 48], [u8; 48]), b: ([u8; 48], [u8; 48], [u8; 48], [u8; 48])) -> Result<[u8; 192], CryptoError> {
        let (pa, pb) = (pad_g2(&a), pad_g2(&b));
        let mut gpu = global().map_err(device_error)?.lock().map_err(device_error)?;
        let (out, st) = gpu.bls12_381_g2_add_batch(&pa, &pb).map_err(device_error)?;
        match st.first().copied() {
            Some(ItemStatus::Ok | ItemStatus::OkIdentity) => Ok(unpad::<192>(&out)),
            Some(bad) => Err(item_error(bad, "G2 point not on curve")),
            None => Err(CryptoError::Other("b200zk returned no status".to_string())),
        }
    }

    fn bls12_381_g2_msm(&self, pairs: &[(([u8; 48], [u8; 48], [u8; 48], [u8; 48]), [u8; 32])]) -> Result<[u8; 192], CryptoError> {
        let mut calldata = Vec::with_capacity(pairs.len().saturating_mul(288));
        for (point, scalar) in pairs {
            calldata.extend_from_slice(&pad_g2(point));
            calldata.extend_from_slice(scalar);
        }
        let mut gpu = global().map_err(device_error)?.lock().map_err(device_error)?;
        let res = gpu.bls12_381_g2_msm_batch(&[calldata.as_slice()]).map_err(device_error)?;
        match res.first() {
            Some(Ok(out)) => Ok(unpad::<192>(out)),
            Some(Err(bad)) => Err(item_error(*bad, "G2 point not on curve or not in subgroup")),
            None => Err(CryptoError::Other("b200zk returned no result".to_string())),
        }
    }
}

/// The trait's 48-byte coordinates -> the EIP-2537 64-byte form the device takes (16 leading zero bytes each).
fn pad_fps<const N: usize>(fps: [&[u8; 48]; N]) -> Vec<u8> {
    let mut out = Vec::with_capacity(64 * N);
    for fp in fps {
        out.extend_from_slice(&[0u8; 16]);
        out.extend_from_slice(fp);
    }
    out
}

fn pad_g1((x, y): &([u8; 48], [u8; 48])) -> Vec<u8> {
    pad_fps([x, y])
}

/// G2 in the trait's and EIP-2537's order: x.c0, x.c1, y.c0, y.c1.
fn pad_g2((x0, x1, y0, y1): &([u8; 48], [u8; 48], [u8; 48], [u8; 48])) -> Vec<u8> {
    pad_fps([x0, x1, y0, y1])
}

/// The device's padded output -> the trait's unpadded form (serialize_bls12_g1 / _g2: 48-byte coordinates in the same
/// order, the identity all zero).  Every 64-byte slot starts with 16 zero bytes, so dropping them loses nothing.
fn unpad<const N: usize>(padded: &[u8]) -> [u8; N] {
    let mut out = [0u8; N];
    for (dst, src) in out.chunks_mut(48).zip(padded.chunks(64)) {
        dst.copy_from_slice(&src[16..64]);
    }
    out
}
